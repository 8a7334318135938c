// epid_find_peaks: pylinac.core.profile.find_peaks (core/profile.py:2545-2649) for one host profile.
#include <cmath>

#include "peaks.cuh"

namespace epid {

constexpr int FP_THREADS = 256;

struct FpOut {
    int count;
    int pad;
};

__global__ void __launch_bounds__(FP_THREADS)
k_find_peaks(const double* __restrict__ x, int n, PeakArgs a, int cap, int* idx, double* prom, int* lb, int* rb, double* wh,
             double* lip, double* rip, int* flag, double* skey, int* sidx, FpOut* out) {
    __shared__ int s_small[FP_THREADS + 8];
    PeakWork w;
    w.cap = cap;
    w.idx = idx; w.prom = prom; w.lbase = lb; w.rbase = rb; w.width_height = wh; w.lip = lip; w.rip = rip;
    w.flag = flag; w.skey = skey; w.sidx = sidx; w.s_small = s_small;
    const int c = block_find_peaks(x, n, a, w);
    if (threadIdx.x == 0) out->count = c;
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_find_peaks(epid_ctx* ctx, const double* values, int32_t n, const epid_peak_params* p, int32_t cap,
                                   int64_t* idx, double* heights, double* prominences, int64_t* left_bases, int64_t* right_bases,
                                   double* widths, double* width_heights, double* left_ips, double* right_ips, int32_t* count) {
    EPID_REQUIRE(ctx && values && p && count, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(n >= 1, EPID_ERR_INVALID, "empty profile");
    // scipy's _peak_widths rejects a negative rel_height before it looks at the peaks, so the reference raises for any profile
    EPID_REQUIRE(!(1.0 - p->fwxm_height < 0.0), EPID_ERR_INVALID, "`rel_height` must be greater or equal to 0.0 (fwxm_height %g > 1)",
                 p->fwxm_height);
    EPID_CUDA(cudaSetDevice(ctx->device));
    // ---- _parse_peak_args (core/profile.py:2626-2649) on the host: needs min/max of the values
    double vmin = values[0], vmax = values[0];
    for (int i = 1; i < n; i++) { vmin = fmin(vmin, values[i]); vmax = fmax(vmax, values[i]); }
    double thr = p->threshold;
    if (thr >= 0.0 && thr <= 1.0) thr = vmin + thr * (vmax - vmin);
    double sep = p->peak_separation;
    if (sep >= 0.0 && sep <= 1.0) { const int s = (int)(sep * (double)n); sep = s > 1 ? s : 1; }
    int lo, hi;
    if (fmax(p->search_lo, p->search_hi) <= 1.0) {
        lo = (int)(p->search_lo * (double)n);
        hi = (int)(p->search_hi * (double)n);
    } else {
        lo = (int)p->search_lo;
        hi = (int)p->search_hi;
    }
    // python slice semantics
    if (lo < 0) lo += n; if (lo < 0) lo = 0; if (lo > n) lo = n;
    if (hi < 0) hi += n; if (hi < 0) hi = 0; if (hi > n) hi = n;
    const int m = hi > lo ? hi - lo : 0;
    *count = 0;
    if (m < 3 || p->max_number == 0) return EPID_OK;   // no interior sample -> no peak; [:0] keeps none
    PeakArgs a;
    a.hmin = thr;
    a.distance = (int)ceil(sep);
    a.pmin = p->required_prominence;
    a.wmin = p->min_width;
    a.rel_height = 1.0 - p->fwxm_height;
    // [:max_number] of the descending order: a negative max_number keeps all but the -max_number smallest, so a first launch
    // counts the peaks and a second keeps count + max_number of them
    const bool drop_smallest = p->max_number < 0 && p->max_number != EPID_PEAKS_ALL;
    a.max_number = p->max_number > 0 ? p->max_number : 0;
    a.sort_by_height = p->peak_sort == 1;
    const int pcap = m / 2 + 1;
    int cap2 = 1;
    while (cap2 < pcap) cap2 <<= 1;
    const size_t bytes = sizeof(double) * (size_t)m + sizeof(double) * (size_t)(4 * pcap + cap2) + sizeof(int) * (size_t)(4 * pcap + cap2) + 4096;
    int rc = ensure_scratch(ctx, bytes);
    if (rc != EPID_OK) return rc;
    char* q = (char*)ctx->scratch;
    auto take = [&](size_t b) { char* r = q; q += (b + 255) / 256 * 256; return r; };
    double* d_x = (double*)take(sizeof(double) * m);
    double* d_prom = (double*)take(sizeof(double) * pcap);
    double* d_wh = (double*)take(sizeof(double) * pcap);
    double* d_lip = (double*)take(sizeof(double) * pcap);
    double* d_rip = (double*)take(sizeof(double) * pcap);
    double* d_skey = (double*)take(sizeof(double) * cap2);
    int* d_idx = (int*)take(sizeof(int) * pcap);
    int* d_lb = (int*)take(sizeof(int) * pcap);
    int* d_rb = (int*)take(sizeof(int) * pcap);
    int* d_flag = (int*)take(sizeof(int) * pcap);
    int* d_sidx = (int*)take(sizeof(int) * cap2);
    FpOut* d_out = (FpOut*)take(sizeof(FpOut));
    if ((size_t)(q - (char*)ctx->scratch) > ctx->scratch_bytes) {
        rc = ensure_scratch(ctx, (size_t)(q - (char*)ctx->scratch));
        if (rc != EPID_OK) return rc;
        return epid_find_peaks(ctx, values, n, p, cap, idx, heights, prominences, left_bases, right_bases, widths, width_heights, left_ips, right_ips, count);
    }
    EPID_CUDA(cudaMemcpyAsync(d_x, values + lo, sizeof(double) * m, cudaMemcpyHostToDevice, ctx->stream));
    FpOut ho;
    for (int pass = 0;; pass++) {
        k_find_peaks<<<1, FP_THREADS, 0, ctx->stream>>>(d_x, m, a, pcap, d_idx, d_prom, d_lb, d_rb, d_wh, d_lip, d_rip, d_flag, d_skey, d_sidx, d_out);
        ctx->launches++;
        EPID_CUDA(cudaMemcpyAsync(&ho, d_out, sizeof(ho), cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaStreamSynchronize(ctx->stream));
        EPID_REQUIRE(ho.count >= 0, EPID_ERR_UNSUPPORTED, "peak capacity exceeded");
        if (!drop_smallest || pass == 1) break;
        a.max_number = ho.count + p->max_number;
        if (a.max_number <= 0) return EPID_OK;
    }
    const int c = ho.count;
    EPID_REQUIRE(c <= cap, EPID_ERR_INVALID, "output capacity %d too small for %d peaks", cap, c);
    std::vector<int> hi_idx(c), hlb(c), hrb(c);
    std::vector<double> hprom(c), hwh(c), hlip(c), hrip(c);
    if (c > 0) {
        EPID_CUDA(cudaMemcpyAsync(hi_idx.data(), d_idx, sizeof(int) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaMemcpyAsync(hlb.data(), d_lb, sizeof(int) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaMemcpyAsync(hrb.data(), d_rb, sizeof(int) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaMemcpyAsync(hprom.data(), d_prom, sizeof(double) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaMemcpyAsync(hwh.data(), d_wh, sizeof(double) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaMemcpyAsync(hlip.data(), d_lip, sizeof(double) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaMemcpyAsync(hrip.data(), d_rip, sizeof(double) * c, cudaMemcpyDeviceToHost, ctx->stream));
        EPID_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    for (int i = 0; i < c; i++) {
        // peak_idxs += shift_amount (core/profile.py:2613); the interpolated positions stay relative to the trimmed array
        if (idx) idx[i] = (int64_t)hi_idx[i] + lo;
        if (heights) heights[i] = values[lo + hi_idx[i]];
        if (prominences) prominences[i] = hprom[i];
        if (left_bases) left_bases[i] = hlb[i];
        if (right_bases) right_bases[i] = hrb[i];
        if (widths) widths[i] = hrip[i] - hlip[i];
        if (width_heights) width_heights[i] = hwh[i];
        if (left_ips) left_ips[i] = hlip[i];
        if (right_ips) right_ips[i] = hrip[i];
    }
    *count = c;
    return EPID_OK;
}
