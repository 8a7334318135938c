// gamma_geometric (reference core/gamma.py:105-226; Ju et al. 2008) and gamma_1d (core/gamma.py:333-460; Low et al. 2004) for a
// ragged batch of profile pairs.  The host normalises, masks, sorts and packs; every pair's evaluation samples and evaluated reference
// points are rows of one CSR layout (eval_off, pt_off).  One upload through page-locked staging, one kernel, one download, one stream
// synchronisation.  -fmad=false: every fma below is written out, where the reference's BLAS dot products round as one.
//
// k_gamma_geometric: a warp per evaluated reference point.  The window is the reference's: argmin |x_eval - (ref_x -+ dta)| widened by
// one sample each side and clamped, with left and right swapped for decreasing x.  The reference subtracts the unnormalised DTA from the
// normalised x, so the half-width is dta in normalised units (dta**2 in the caller's units); this kernel does the same.  Lanes take the
// window's segments, segment_distance (gamma1d.cuh) gives each distance, and the reduction is Python's min(): nan iff the first
// segment's distance is nan, else the least non-nan one; then min(that, cap) likewise.
//
// k_gamma1d: a warp per evaluated reference point, lanes over its num samples of np.linspace(ref_x - dta, ref_x + dta, num), each
// interpolated as scipy's interp1d(kind="linear", fill_value="extrapolate") does, then sqrt(dist**2 / dta**2 + dose**2 / dose_ta**2)
// with the same min() rules.  The squares are correctly rounded products.
#include <algorithm>

#include "common.cuh"
#include "gamma1d.cuh"

namespace epid {
namespace {

constexpr int kWarps = 8;

__device__ __forceinline__ int pair_of(const long long* __restrict__ pt_off, int n, long long pt) {
    int lo = 0, hi = n;                  // last pair whose first point is <= pt
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (pt_off[mid] <= pt) lo = mid; else hi = mid;
    }
    return lo;
}

// Python's min() of the lane values in visiting order: first_nan from the lane holding the first item, the rest a nan-skipping min
__device__ __forceinline__ double py_min_warp(double m, bool first_nan_here, bool has_first) {
    for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
    const unsigned fn = __ballot_sync(0xffffffffu, has_first && first_nan_here);
    return fn ? (double)NAN : m;
}

__global__ void __launch_bounds__(kWarps * 32) k_gamma_geometric(
    int n, long long n_pts, const long long* __restrict__ eval_off, const long long* __restrict__ pt_off, const int* __restrict__ dec,
    const double* __restrict__ ex, const double* __restrict__ ey, const double* __restrict__ rx, const double* __restrict__ ry,
    double dta, double cap, double* __restrict__ gamma, int* __restrict__ svd_fail) {
    const long long pt = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pt >= n_pts) return;
    const int f = pair_of(pt_off, n, pt);
    const double* x = ex + eval_off[f];
    const double* y = ey + eval_off[f];
    const int m = (int)(eval_off[f + 1] - eval_off[f]);
    const bool d = dec[f] != 0;
    const double px = rx[pt], py = ry[pt];
    double tl = px - dta, tr = px + dta;
    if (d) {
        const double t = tl;
        tl = tr;
        tr = t;
    }
    const int left = max(g1::argmin_abs(x, m, tl, d) - 1, 0);
    const int right = min(g1::argmin_abs(x, m, tr, d) + 1, m - 1);
    double best = NAN;
    bool first_nan = false, fail = false;
    for (int j = left + lane; j < right; j += 32) {
        const double v = g1::segment_distance(px, py, x[j], y[j], x[j + 1], y[j + 1], &fail);
        if (j == left) first_nan = isnan(v);
        best = fmin(best, v);
    }
    const double g = py_min_warp(best, first_nan, lane == 0);
    if (__any_sync(0xffffffffu, fail)) {
        if (lane == 0) svd_fail[f] = 1;
    }
    if (lane == 0) gamma[pt] = cap < g ? cap : g;
}

// numpy's ordering for searchsorted: nan sorts last
__device__ __forceinline__ bool np_lt(double a, double b) { return a < b || (isnan(b) && !isnan(a)); }

__global__ void __launch_bounds__(kWarps * 32) k_gamma1d(
    int n, long long n_pts, const long long* __restrict__ eval_off, const long long* __restrict__ pt_off, const int* __restrict__ f32,
    const double* __restrict__ ex, const double* __restrict__ ey, const double* __restrict__ rx, const double* __restrict__ ry,
    const double* __restrict__ dose_ta2, double dta, double dta2, int num, double cap, double* __restrict__ gamma,
    double* __restrict__ samples, double* __restrict__ sample_x) {
    const long long pt = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pt >= n_pts) return;
    const int f = pair_of(pt_off, n, pt);
    const double* x = ex + eval_off[f];
    const double* y = ey + eval_off[f];
    const int m = (int)(eval_off[f + 1] - eval_off[f]);
    const bool single = f32[f] != 0;
    const double px = rx[pt], py = ry[pt], dd2 = dose_ta2[pt];
    // np.linspace(start, stop, num): i * step + start, or (i / div) * delta + start when the step underflows to 0; the last sample is stop
    const double start = px - dta, stop = px + dta, delta = stop - start;
    const int div = num - 1;
    const double step = div > 0 ? delta / div : 0.0;
    double best = NAN;
    bool first_nan = false;
    for (int k = lane; k < num; k += 32) {
        double xs;
        if (div <= 0) xs = 0.0 * delta + start;
        else if (k == div) xs = stop;
        else if (step == 0.0) xs = ((double)k / div) * delta + start;
        else xs = (double)k * step + start;
        int lo = 0, hi = m;              // searchsorted(x, xs, side="left"), clipped to [1, m - 1]
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (np_lt(x[mid], xs)) lo = mid + 1; else hi = mid;
        }
        const int i = min(max(lo, 1), m - 1), il = i > 0 ? i - 1 : m - 1;      // one sample: numpy's x[-1] is x[0]
        const double xl = x[il], xh = x[i], w = xh - xl;
        const double v = ((xs - xl) / w) * y[i] + ((xh - xs) / w) * y[il];
        const size_t o = (size_t)pt * num + k;
        samples[o] = v;
        sample_x[o] = xs;
        const double dist = fabs(px - xs), dose = py - v;
        const double t2 = single ? (double)((float)(dose * dose) / (float)dd2) : dose * dose / dd2;
        const double cg = sqrt(dist * dist / dta2 + t2);
        if (k == 0) first_nan = isnan(cg);
        best = fmin(best, cg);
    }
    const double g = py_min_warp(best, first_nan, lane == 0);
    if (lane == 0) gamma[pt] = cap < g ? cap : g;
}

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

// Packs `parts` into page-locked staging and one device allocation: one upload.  Returns the device address of each part.
struct Packed {
    std::vector<size_t> at;
    size_t bytes = 0;
};

Packed layout(const std::vector<size_t>& sizes) {
    Packed p;
    for (size_t s : sizes) {
        p.at.push_back(p.bytes);
        p.bytes += al256(s);
    }
    return p;
}

}  // namespace
}  // namespace epid

using namespace epid;

namespace {

// inputs: {pointer, bytes} in order; outputs: {pointer, bytes}; run(device addresses of inputs then outputs) enqueues the kernel
template <class Launch>
int gamma1d_call(epid_ctx* ctx, const std::vector<std::pair<const void*, size_t>>& in, const std::vector<std::pair<void*, size_t>>& out,
                 Launch launch, const char* what) {
    std::vector<size_t> in_sz, out_sz;
    for (auto& p : in) in_sz.push_back(p.second);
    for (auto& p : out) out_sz.push_back(p.second);
    const Packed li = layout(in_sz), lo = layout(out_sz);
    EPID_CUDA(cudaSetDevice(ctx->device));
    int rc = ensure_scratch(ctx, li.bytes + lo.bytes);
    if (rc == EPID_OK) rc = ensure_pinned(ctx, std::max(li.bytes, lo.bytes));
    if (rc != EPID_OK) return rc;
    char* h = (char*)ctx->pinned;
    char* d = (char*)ctx->scratch;
    cudaStream_t s = ctx->stream;
    EPID_CUDA(cudaStreamSynchronize(s));                  // the staging buffer may still feed an earlier copy
    for (size_t i = 0; i < in.size(); i++)
        if (in[i].second) std::memcpy(h + li.at[i], in[i].first, in[i].second);
    EPID_CUDA(cudaMemcpyAsync(d, h, li.bytes, cudaMemcpyHostToDevice, s));
    std::vector<char*> dev;
    for (size_t a : li.at) dev.push_back(d + a);
    for (size_t a : lo.at) dev.push_back(d + li.bytes + a);
    rc = launch(dev, s);
    if (rc != EPID_OK) return rc;
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h, d + li.bytes, lo.bytes, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        set_error("%s failed: %s", what, cudaGetErrorString(e));
        return EPID_ERR_CUDA;
    }
    for (size_t i = 0; i < out.size(); i++)
        if (out[i].second) std::memcpy(out[i].first, h + lo.at[i], out[i].second);
    return EPID_OK;
}

int check_offsets(int32_t n, const int64_t* eval_off, const int64_t* pt_off, int min_eval) {
    EPID_REQUIRE(eval_off[0] == 0 && pt_off[0] == 0, EPID_ERR_INVALID, "offsets must start at 0");
    for (int i = 0; i < n; i++) {
        const int64_t m = eval_off[i + 1] - eval_off[i], p = pt_off[i + 1] - pt_off[i];
        EPID_REQUIRE(p >= 0 && m <= INT32_MAX, EPID_ERR_INVALID, "pair %d: bad offsets", i);
        EPID_REQUIRE(p == 0 || m >= min_eval, EPID_ERR_INVALID, "pair %d: %lld evaluation samples, need %d", i, (long long)m, min_eval);
    }
    return EPID_OK;
}

}  // namespace

extern "C" int32_t epid_gamma_geometric(epid_ctx* ctx, int32_t n, const int64_t* eval_off, const int64_t* pt_off, const int32_t* decreasing,
                                        const double* eval_x, const double* eval_y, const double* ref_x, const double* ref_y, double dta,
                                        double cap, double* gamma, int32_t* svd_fail) {
    EPID_REQUIRE(ctx && n > 0 && eval_off && pt_off && decreasing && gamma && svd_fail, EPID_ERR_INVALID, "NULL argument");
    int rc = check_offsets(n, eval_off, pt_off, 2);
    if (rc != EPID_OK) return rc;
    const long long ne = eval_off[n], np_ = pt_off[n];
    std::fill(svd_fail, svd_fail + n, 0);
    if (np_ == 0) return EPID_OK;
    return gamma1d_call(
        ctx,
        {{eval_off, 8 * (size_t)(n + 1)}, {pt_off, 8 * (size_t)(n + 1)}, {decreasing, 4 * (size_t)n}, {eval_x, 8 * (size_t)ne}, {eval_y, 8 * (size_t)ne}, {ref_x, 8 * (size_t)np_}, {ref_y, 8 * (size_t)np_}},
        {{gamma, 8 * (size_t)np_}, {svd_fail, 4 * (size_t)n}},
        [&](const std::vector<char*>& a, cudaStream_t s) {
            EPID_CUDA(cudaMemsetAsync(a[8], 0, 4 * (size_t)n, s));
            k_gamma_geometric<<<(unsigned)((np_ + kWarps - 1) / kWarps), kWarps * 32, 0, s>>>(
                n, np_, (const long long*)a[0], (const long long*)a[1], (const int*)a[2], (const double*)a[3], (const double*)a[4],
                (const double*)a[5], (const double*)a[6], dta, cap, (double*)a[7], (int*)a[8]);
            return EPID_OK;
        },
        "k_gamma_geometric");
}

extern "C" int32_t epid_gamma1d(epid_ctx* ctx, int32_t n, const int64_t* eval_off, const int64_t* pt_off, const int32_t* dose_f32,
                                const double* eval_x, const double* eval_y, const double* ref_x, const double* ref_y, const double* dose_ta2,
                                double dta, double dta2, int32_t num, double cap, double* gamma, double* samples, double* sample_x) {
    EPID_REQUIRE(ctx && n > 0 && eval_off && pt_off && dose_f32 && gamma && samples && sample_x, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(num >= 1, EPID_ERR_INVALID, "num = %d samples per point, need at least 1", num);
    int rc = check_offsets(n, eval_off, pt_off, 1);
    if (rc != EPID_OK) return rc;
    const long long ne = eval_off[n], np_ = pt_off[n];
    if (np_ == 0) return EPID_OK;
    const size_t ns = 8 * (size_t)np_ * num;
    return gamma1d_call(
        ctx,
        {{eval_off, 8 * (size_t)(n + 1)}, {pt_off, 8 * (size_t)(n + 1)}, {dose_f32, 4 * (size_t)n}, {eval_x, 8 * (size_t)ne},
         {eval_y, 8 * (size_t)ne}, {ref_x, 8 * (size_t)np_}, {ref_y, 8 * (size_t)np_}, {dose_ta2, 8 * (size_t)np_}},
        {{gamma, 8 * (size_t)np_}, {samples, ns}, {sample_x, ns}},
        [&](const std::vector<char*>& a, cudaStream_t s) {
            k_gamma1d<<<(unsigned)((np_ + kWarps - 1) / kWarps), kWarps * 32, 0, s>>>(
                n, np_, (const long long*)a[0], (const long long*)a[1], (const int*)a[2], (const double*)a[3], (const double*)a[4],
                (const double*)a[5], (const double*)a[6], (const double*)a[7], dta, dta2, num, cap, (double*)a[8], (double*)a[9],
                (double*)a[10]);
            return EPID_OK;
        },
        "k_gamma1d");
}
