// Frame statistics of uint16 frame views: min, max, sum, row sums, column sums, the four check_inversion corner sums and EXACT order
// statistics from a 65536-bin histogram.
//
// Replaces the reference's numpy passes: array.min()/max() (picketfence.py:231-232, core/image.py:851),
// np.percentile / np.median of the full frame (picketfence.py:233,1510; core/image.py:918-920),
// np.mean(image, axis) (picketfence.py:748-750), corner means (core/image.py:881-896).
#include "stats.cuh"

namespace epid {

int make_stats_geom(StatsGeom* g, int H, int W) {
    if (H <= 0 || W <= 0 || H > STATS_MAX_DIM || W > STATS_MAX_DIM) {
        set_error("frame view %d x %d outside the supported range (1..%d)", H, W, STATS_MAX_DIM);
        return EPID_ERR_UNSUPPORTED;
    }
    memset(g, 0, sizeof(*g));
    g->H = H;
    g->W = W;
    const int vpr = (W + 7 + 7) / 8;  // worst-case misalignment of 7 pixels
    g->vprp = (vpr + 31) / 32 * 32;
    g->groups = STATS_THREADS / g->vprp;
    if (g->groups < 1) {
        set_error("frame view too wide (%d)", W);
        return EPID_ERR_UNSUPPORTED;
    }
    return EPID_OK;
}

__global__ void k_refs_from_batch(const uint16_t* base, int n, int H0, int W0, int r0, int c0, FrameRef* refs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    refs[i].origin = base + (size_t)i * H0 * W0 + (size_t)r0 * W0 + c0;
    refs[i].pitch = W0;
    refs[i].pad = 0;
}

void launch_refs_from_batch(epid_ctx* ctx, cudaStream_t stream, const uint16_t* base, int n, int H0, int W0, int r0, int c0, FrameRef* refs) {
    k_refs_from_batch<<<(n + 127) / 128, 128, 0, stream>>>(base, n, H0, W0, r0, c0, refs);
    ctx->launches++;
}

// ------------------------------------------------------------------------------------------------ exact histogram path
// k_hist_view spreads a frame over HV_PARTS CTAs of row blocks, and a view wider than HV_STRIP columns over column strips as well: each
// CTA streams its rows of its strip with 16-byte loads, counts every pixel through the bin cache of stats.cuh into the frame's global
// histogram, keeps column sums in registers and writes row sums (accumulates them, when there are several strips).  k_stats_from_hist,
// one CTA per frame, turns the 65536-bin histogram into min / max / sum / order statistics and adds the column partials.  32-bit
// counters throughout.
constexpr int HV_PARTS = 16;
constexpr int HV_THREADS = 256;
constexpr int HV_WARPS = HV_THREADS / 32;
// columns of a strip: with the worst misalignment of 7 pixels they fill the 256 vectors of k_hist_view<8>; a multiple of 8, so every
// strip keeps the view's 16-byte phase
constexpr int HV_STRIP = 2040;

template <int VPL>
__global__ void __launch_bounds__(HV_THREADS)
k_hist_view(const StatsGeom g, const FrameRef* __restrict__ frames, uint32_t* __restrict__ hist, uint32_t* __restrict__ rowsum_out,
            uint32_t* __restrict__ colpart, int wa) {
    __shared__ HistCache s_cache;
    extern __shared__ uint32_t s_col[];      // wa column accumulators of the CTA
    const int fi = blockIdx.y, strip = blockIdx.x / HV_PARTS, part = blockIdx.x - strip * HV_PARTS;
    const int nstrips = gridDim.x / HV_PARTS;
    const FrameRef fr = frames[fi];
    const uint16_t* __restrict__ f = fr.origin + strip * HV_STRIP;
    const int W = min(g.W - strip * HV_STRIP, HV_STRIP);
    const int pitch = fr.pitch;
    uint32_t* h = hist + (size_t)fi * 65536;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const bool aligned = (pitch % 8) == 0;
    const int mis = aligned ? (int)((reinterpret_cast<uintptr_t>(f) >> 1) & 7) : 0;
    hist_cache_init(s_cache);
    for (int i = tid; i < wa; i += HV_THREADS) s_col[i] = 0;
    __syncthreads();
    const int rp = (g.H + HV_PARTS - 1) / HV_PARTS;
    const int r0 = part * rp, r1 = min(g.H, r0 + rp);
    uint32_t csum[VPL][8];
#pragma unroll
    for (int k = 0; k < VPL; k++)
#pragma unroll
        for (int e = 0; e < 8; e++) csum[k][e] = 0;
    for (int r = r0 + wid; r < r1; r += HV_WARPS) {
        const uint16_t* rowp = f + (size_t)r * pitch;
        uint32_t rs = 0;
        uint4 q[VPL];
        uint32_t valid[VPL];
#pragma unroll
        for (int k = 0; k < VPL; k++) {
            const int col_first = (lane + 32 * k) * 8 - mis;
            uint32_t vm = 0;
#pragma unroll
            for (int e = 0; e < 8; e++) { const int cidx = col_first + e; if (cidx >= 0 && cidx < W) vm |= 1u << e; }
            valid[k] = vm;
            q[k] = make_uint4(0, 0, 0, 0);
            if (vm) {
                if (aligned) q[k] = ldg_stream16(rowp + col_first);
                else {
                    uint32_t w4[4] = {0, 0, 0, 0};
#pragma unroll
                    for (int e = 0; e < 8; e++) if (vm >> e & 1) w4[e >> 1] |= (uint32_t)__ldg(rowp + col_first + e) << ((e & 1) * 16);
                    q[k] = make_uint4(w4[0], w4[1], w4[2], w4[3]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < VPL; k++) {
            const uint32_t w4[4] = {q[k].x, q[k].y, q[k].z, q[k].w};
            const bool any = __any_sync(0xffffffffu, valid[k] != 0);
            if (!any) continue;     // warp-uniform
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const uint32_t v = (w4[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
                const bool in = valid[k] >> e & 1;
                hist_cache_add(s_cache, h, v, in);
                if (in) { csum[k][e] += v; rs += v; }
            }
        }
        rs = warp_sum(rs);
        if (lane == 0 && rowsum_out) {
            if (nstrips > 1) atomicAdd(&rowsum_out[(size_t)fi * g.H + r], rs);
            else rowsum_out[(size_t)fi * g.H + r] = rs;
        }
    }
    // column partials: registers -> CTA accumulators -> one partial row per (frame, part), wa columns per strip
#pragma unroll
    for (int k = 0; k < VPL; k++)
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int ac = (lane + 32 * k) * 8 + e;
            if (ac < wa && csum[k][e]) atomicAdd(&s_col[ac], csum[k][e]);
        }
    __syncthreads();
    if (colpart)
        for (int i = tid; i < wa; i += HV_THREADS) colpart[((size_t)fi * HV_PARTS + part) * nstrips * wa + strip * wa + i] = s_col[i];
    hist_cache_flush(s_cache, h);
}

__global__ void __launch_bounds__(HIST_RANK_THREADS)
k_stats_from_hist(const StatsGeom g, const FrameRef* __restrict__ frames, const uint32_t* __restrict__ hist, const uint32_t* __restrict__ colpart,
                  int wa, FrameStats* __restrict__ stats, uint32_t* __restrict__ colsum_out) {
    __shared__ HistRanks s;
    __shared__ unsigned long long s_wsum[HIST_RANK_THREADS];
    __shared__ unsigned long long s_corner;
    const int fi = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const FrameRef fr = frames[fi];
    if (tid == 0) s_corner = 0;
    hist_rank_search(hist + (size_t)fi * 65536, g.ranks, g.nranks, s, s_wsum);
    // corner boxes (core/image.py:881-894)
    if (g.box > 0) {
        const int per = g.box * g.box;
        unsigned long long cs = 0;
        for (int i = tid; i < 4 * per; i += HIST_RANK_THREADS) {
            const int b = i / per, o = i - b * per;
            const int y = o / g.box, x = o - y * g.box;
            const int rr = ((b & 2) ? g.H - g.rp - g.box : g.rp) + y;
            const int cc = ((b & 1) ? g.W - g.cp - g.box : g.cp) + x;
            if (rr >= 0 && rr < g.H && cc >= 0 && cc < g.W) cs += __ldg(fr.origin + (size_t)rr * fr.pitch + cc);
        }
        cs = warp_sum(cs);
        if (lane == 0 && cs) atomicAdd(&s_corner, cs);
    }
    // column sums: the parts' partial rows (vector-grid columns of each strip) -> view columns
    if (colsum_out && colpart) {
        const bool aligned = (fr.pitch % 8) == 0;
        const int mis = aligned ? (int)((reinterpret_cast<uintptr_t>(fr.origin) >> 1) & 7) : 0;
        const int row = (g.W + HV_STRIP - 1) / HV_STRIP * wa;
        for (int x = tid; x < g.W; x += HIST_RANK_THREADS) {
            const int strip = x / HV_STRIP;
            const int ac = strip * wa + (x - strip * HV_STRIP) + mis;
            uint32_t sum = 0;
            for (int p = 0; p < HV_PARTS; p++) sum += colpart[((size_t)fi * HV_PARTS + p) * row + ac];
            colsum_out[(size_t)fi * g.W + x] = sum;
        }
    }
    __syncthreads();
    if (tid == 0) {
        unsigned long long tot = 0;
        for (int k = 0; k < HIST_RANK_THREADS; k++) tot += s_wsum[k];
        FrameStats& o = stats[fi];
        o.mn = s.first;
        o.mx = s.last;
        o.npix = (uint32_t)g.H * (uint32_t)g.W;
        o.sum = tot;
        o.corner_sum = s_corner;
        o.inv_certified = 0;
        for (int qi = 0; qi < g.nranks; qi++) o.ostat[qi] = s.values[qi];
    }
}

static int ensure_hist_scratch(epid_ctx* ctx, size_t bytes) {
    if (ctx->hist_bytes >= bytes) return EPID_OK;
    if (ctx->hist_scratch) { EPID_CUDA(cudaStreamSynchronize(ctx->stream)); EPID_CUDA(cudaFree(ctx->hist_scratch)); ctx->hist_scratch = nullptr; ctx->hist_bytes = 0; }
    cudaError_t e = cudaMalloc(&ctx->hist_scratch, bytes);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); return EPID_ERR_NOMEM; }
    ctx->hist_bytes = bytes;
    return EPID_OK;
}

// launch shape of k_hist_view for views of W columns
struct HvShape {
    int strips;      // column strips of HV_STRIP columns
    int vpl;         // vectors per lane
    int wa;          // columns of a strip's vector grid
};

static HvShape hv_shape(int W) {
    const int sw = W < HV_STRIP ? W : HV_STRIP;
    const int vpl = ((sw + 7 + 7) / 8 + 31) / 32;
    return {(W + HV_STRIP - 1) / HV_STRIP, vpl, vpl * 32 * 8};
}

// wa = 0: no column sums
static void launch_hist_view(cudaStream_t stream, const StatsGeom& g, const HvShape& hv, const FrameRef* d_frames, int cn, uint32_t* hist,
                             uint32_t* rowsum, uint32_t* colpart, int wa) {
    const dim3 grid(HV_PARTS * hv.strips, cn);
    const size_t smem = sizeof(uint32_t) * wa;
    if (hv.vpl <= 4) k_hist_view<4><<<grid, HV_THREADS, smem, stream>>>(g, d_frames, hist, rowsum, colpart, wa);
    else k_hist_view<8><<<grid, HV_THREADS, smem, stream>>>(g, d_frames, hist, rowsum, colpart, wa);
}

int launch_frame_stats(epid_ctx* ctx, cudaStream_t stream, const StatsGeom& g, const FrameRef* d_frames, int n, FrameStats* d_stats,
                       uint32_t* d_rowsum, uint32_t* d_colsum) {
    const HvShape hv = hv_shape(g.W);
    const int chunk = n < 256 ? n : 256;
    const size_t hist_b = sizeof(uint32_t) * (size_t)chunk * 65536;
    const size_t col_b = sizeof(uint32_t) * (size_t)chunk * HV_PARTS * hv.strips * hv.wa;
    int rc = ensure_hist_scratch(ctx, hist_b + col_b + 512);
    if (rc != EPID_OK) return rc;
    uint32_t* hist = (uint32_t*)ctx->hist_scratch;
    uint32_t* colpart = d_colsum ? (uint32_t*)((char*)ctx->hist_scratch + (hist_b + 255) / 256 * 256) : nullptr;
    for (int c0 = 0; c0 < n; c0 += chunk) {
        const int cn = n - c0 < chunk ? n - c0 : chunk;
        EPID_CUDA(cudaMemsetAsync(hist, 0, sizeof(uint32_t) * (size_t)cn * 65536, stream));
        uint32_t* rs = d_rowsum ? d_rowsum + (size_t)c0 * g.H : nullptr;
        if (rs && hv.strips > 1) EPID_CUDA(cudaMemsetAsync(rs, 0, sizeof(uint32_t) * (size_t)cn * g.H, stream));
        launch_hist_view(stream, g, hv, d_frames + c0, cn, hist, rs, colpart, hv.wa);
        k_stats_from_hist<<<cn, HIST_RANK_THREADS, 0, stream>>>(g, d_frames + c0, hist, colpart, hv.wa, d_stats + c0,
                                                                d_colsum ? d_colsum + (size_t)c0 * g.W : nullptr);
        ctx->launches += 2;
        EPID_CUDA(cudaGetLastError());
    }
    return EPID_OK;
}

int launch_frame_histogram(epid_ctx* ctx, cudaStream_t stream, const StatsGeom& g, const FrameRef* d_frames, int n, uint32_t* d_hist) {
    EPID_CUDA(cudaMemsetAsync(d_hist, 0, sizeof(uint32_t) * (size_t)n * 65536, stream));
    launch_hist_view(stream, g, hv_shape(g.W), d_frames, n, d_hist, nullptr, nullptr, 0);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

// ------------------------------------------------------------------------------------------------ certified inversion statistics
// check_inversion_by_histogram (core/image.py:899-926) needs three percentiles of the frame only to DECIDE |p_mid - p_low| >
// |p_mid - p_high|.  Per-pixel histogram atomics bound the exact path by the shared-memory atomic rate, so FieldAnalysis / Starshot
// get the decision from counts instead, the way pf_stream.cu certifies PicketFence's decisions:
//   k_inv_pilot   CTA per frame: 4096-pixel grid sample, 16-step value bisection -> for each percentile a bracket [tL, tU] of sample order
//                 statistics 5 sigma either side of the rank
//   k_inv_stream  IV_PARTS CTAs per frame, one 16-byte load per lane and vector: exact min / max / sum, row sums, column partials and the
//                 six exact counts #(v < T) by packed u16x2 arithmetic (no atomics in the pixel loop)
//   k_inv_finish  CTA per frame: combines the parts; #(v < tL) <= rank_prev and #(v <= tU) > rank_next PROVE tL <= percentile <= tU; if the
//                 resulting intervals of the two distances do not overlap the decision is certified (FrameStats.inv_certified = 2 +
//                 inverted), otherwise the frame is listed for the exact histogram path (ostat exact, inv_certified = 0).
constexpr int IV_PARTS = 16;
constexpr int IV_THREADS = 256;
constexpr int IV_WARPS = IV_THREADS / 32;
constexpr int IV_SAMPLE_ROWS = 16;

struct InvPart {                 // per (frame, part)
    uint32_t cnt[6];
    uint32_t mn, mx;
    unsigned long long total;
};

__global__ void __launch_bounds__(IV_THREADS)
k_inv_pilot(const StatsGeom g, const FrameRef* __restrict__ frames, uint32_t* __restrict__ thr) {
    __shared__ uint32_t b_lo[6], b_hi[6], b_rank[6], b_fix[6];
    __shared__ uint32_t s_cnt[6][IV_WARPS];
    const int fi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const FrameRef fr = frames[fi];
    const int H = g.H, W = g.W;
    const double npix = (double)H * (double)W;
    const uint32_t S = IV_THREADS * IV_SAMPLE_ROWS;
    uint32_t sv[IV_SAMPLE_ROWS];
    {
        const int col = min(W - 1, (int)(((2LL * tid + 1) * W) / (2 * IV_THREADS)));
#pragma unroll
        for (int i = 0; i < IV_SAMPLE_ROWS; i++) {
            const int row = min(H - 1, (int)(((2LL * i + 1) * H) / (2 * IV_SAMPLE_ROWS)));
            sv[i] = __ldg(fr.origin + (size_t)row * fr.pitch + col);
        }
    }
    if (tid < 6) {
        // lower (even) / upper (odd) sample rank of the bracket: 5 sigma of the binomial sample count around the pixel rank's quantile
        const double q = (double)g.ranks[tid] / npix;
        const double sg = sqrt(q * (1.0 - q) * (double)S);
        const double ctr = q * (double)S;
        const double rr = (tid & 1) ? ctr + 5.0 * sg + 3.0 : ctr - 5.0 * sg - 3.0;
        b_fix[tid] = 0;
        if (rr < 0.0) b_fix[tid] = 1;                      // bracket reaches below the sample: tL = 0
        if (rr > (double)(S - 1)) b_fix[tid] = 2;          // above the sample: tU = 65535
        b_rank[tid] = (uint32_t)fmin(fmax(rr, 0.0), (double)(S - 1));
        b_lo[tid] = 0;
        b_hi[tid] = 65535u;
    }
    __syncthreads();
    // smallest value t with #(sample <= t) > rank = the sample's order statistic, by bisection on the value
    for (int step = 0; step < 16; step++) {
        uint32_t c[6];
#pragma unroll
        for (int t = 0; t < 6; t++) {
            const uint32_t mid = (b_lo[t] + b_hi[t]) >> 1;
            uint32_t cc = 0;
#pragma unroll
            for (int i = 0; i < IV_SAMPLE_ROWS; i++) cc += sv[i] <= mid ? 1u : 0u;
            c[t] = warp_sum(cc);
        }
        if (lane == 0) {
#pragma unroll
            for (int t = 0; t < 6; t++) s_cnt[t][wid] = c[t];
        }
        __syncthreads();
        if (tid < 6) {
            uint32_t tot = 0;
            for (int k = 0; k < IV_WARPS; k++) tot += s_cnt[tid][k];
            const uint32_t mid = (b_lo[tid] + b_hi[tid]) >> 1;
            if (tot > b_rank[tid]) b_hi[tid] = mid; else b_lo[tid] = mid + 1;
        }
        __syncthreads();
    }
    if (tid < 6) {
        uint32_t v = b_hi[tid];
        if (b_fix[tid] == 1) v = 0;
        if (b_fix[tid] == 2) v = 65535u;
        // even: T = tL (count of v < tL); odd: T = tU + 1 (count of v <= tU), 65536 = every pixel
        thr[fi * 6 + tid] = (tid & 1) ? v + 1u : v;
    }
}

template <int VPL, bool COLS>
__global__ void __launch_bounds__(IV_THREADS, COLS ? 2 : 3)
k_inv_stream(const StatsGeom g, const FrameRef* __restrict__ frames, const uint32_t* __restrict__ thr, InvPart* __restrict__ parts,
             uint32_t* __restrict__ rowsum_out, uint32_t* __restrict__ colpart, int wa) {
    extern __shared__ uint32_t s_col[];      // wa column accumulators of the CTA (COLS)
    __shared__ uint32_t s_red[IV_WARPS][8];
    __shared__ unsigned long long s_tot[IV_WARPS];
    const int fi = blockIdx.y, part = blockIdx.x;
    const FrameRef fr = frames[fi];
    const uint16_t* __restrict__ f = fr.origin;
    const int pitch = fr.pitch;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const bool aligned = (pitch % 8) == 0;
    const int mis = aligned ? (int)((reinterpret_cast<uintptr_t>(f) >> 1) & 7) : 0;
    if (COLS) { for (int i = tid; i < wa; i += IV_THREADS) s_col[i] = 0; }
    uint32_t T2[6];
#pragma unroll
    for (int t = 0; t < 6; t++) { const uint32_t T = min(thr[fi * 6 + t], 65535u); T2[t] = T | (T << 16); }
    // validity of the lane's vectors is the same for every row: masks of the pixels inside the view
    uint32_t vmask[VPL][4];
    bool anyv[VPL];
#pragma unroll
    for (int k = 0; k < VPL; k++) {
        const int col_first = (lane + 32 * k) * 8 - mis;
        anyv[k] = false;
#pragma unroll
        for (int h2 = 0; h2 < 4; h2++) {
            uint32_t m = 0;
            if (col_first + 2 * h2 >= 0 && col_first + 2 * h2 < g.W) m |= 0xffffu;
            if (col_first + 2 * h2 + 1 >= 0 && col_first + 2 * h2 + 1 < g.W) m |= 0xffff0000u;
            vmask[k][h2] = m;
            anyv[k] = anyv[k] || m != 0;
        }
    }
    const int rp = (g.H + IV_PARTS - 1) / IV_PARTS;
    const int r0 = part * rp, r1 = min(g.H, r0 + rp);
    uint32_t cnt[6] = {0, 0, 0, 0, 0, 0};
    uint32_t mn2 = 0xffffffffu, mx2 = 0;
    unsigned long long total = 0;
    uint32_t csum[COLS ? VPL : 1][8];
    if (COLS) {
#pragma unroll
        for (int k = 0; k < VPL; k++)
#pragma unroll
            for (int e = 0; e < 8; e++) csum[k][e] = 0;
    }
    for (int r = r0 + wid; r < r1; r += IV_WARPS) {
        const uint16_t* rowp = f + (size_t)r * pitch;
        uint4 q[VPL];
#pragma unroll
        for (int k = 0; k < VPL; k++) {
            q[k] = make_uint4(0, 0, 0, 0);
            if (anyv[k]) {
                const int col_first = (lane + 32 * k) * 8 - mis;
                if (aligned) q[k] = ldg_stream16(rowp + col_first);
                else {
                    uint32_t w4[4] = {0, 0, 0, 0};
#pragma unroll
                    for (int e = 0; e < 8; e++)
                        if ((vmask[k][e >> 1] >> ((e & 1) * 16)) & 1u) w4[e >> 1] |= (uint32_t)__ldg(rowp + col_first + e) << ((e & 1) * 16);
                    q[k] = make_uint4(w4[0], w4[1], w4[2], w4[3]);
                }
            }
        }
        uint32_t rs = 0;
#pragma unroll
        for (int k = 0; k < VPL; k++) {
            if (!anyv[k]) continue;
            const uint32_t w4[4] = {q[k].x, q[k].y, q[k].z, q[k].w};
#pragma unroll
            for (int h2 = 0; h2 < 4; h2++) {
                const uint32_t lo = w4[h2] & vmask[k][h2];         // outside the view: 0     (maximum, sums)
                const uint32_t hi = w4[h2] | ~vmask[k][h2];        // outside the view: 65535 (minimum, counts: never < T)
                mn2 = __vminu2(mn2, hi);
                mx2 = __vmaxu2(mx2, lo);
                rs = __dp2a_lo(lo, 0x0101u, rs);
#pragma unroll
                for (int t = 0; t < 6; t++) cnt[t] = __dp2a_lo(__vminu2(__vmaxu2(hi, T2[t]) - hi, 0x00010001u), 0x0101u, cnt[t]);
                if (COLS) {
                    csum[k][2 * h2] = __dp2a_lo(lo, 0x0001u, csum[k][2 * h2]);
                    csum[k][2 * h2 + 1] = __dp2a_lo(lo, 0x0100u, csum[k][2 * h2 + 1]);
                }
            }
        }
        rs = warp_sum(rs);
        total += rs;
        if (lane == 0 && rowsum_out) rowsum_out[(size_t)fi * g.H + r] = rs;
    }
    if (COLS) {
#pragma unroll
        for (int k = 0; k < VPL; k++)
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const int ac = (lane + 32 * k) * 8 + e;
                if (ac < wa && csum[k][e]) atomicAdd(&s_col[ac], csum[k][e]);
            }
    }
    uint32_t mn = min(mn2 & 0xffffu, mn2 >> 16), mx = max(mx2 & 0xffffu, mx2 >> 16);
    mn = warp_min(mn);
    mx = warp_max(mx);
#pragma unroll
    for (int t = 0; t < 6; t++) cnt[t] = warp_sum(cnt[t]);
    if (lane == 0) {
#pragma unroll
        for (int t = 0; t < 6; t++) s_red[wid][t] = cnt[t];
        s_red[wid][6] = mn;
        s_red[wid][7] = mx;
        s_tot[wid] = total;          // every lane holds the warp's row sums
    }
    __syncthreads();
    if (COLS && colpart) for (int i = tid; i < wa; i += IV_THREADS) colpart[((size_t)fi * IV_PARTS + part) * wa + i] = s_col[i];
    if (tid == 0) {
        InvPart o;
        for (int t = 0; t < 6; t++) o.cnt[t] = 0;
        o.mn = 0xffffu; o.mx = 0; o.total = 0;
        for (int k = 0; k < IV_WARPS; k++) {
            for (int t = 0; t < 6; t++) o.cnt[t] += s_red[k][t];
            o.mn = min(o.mn, s_red[k][6]);
            o.mx = max(o.mx, s_red[k][7]);
            o.total += s_tot[k];
        }
        parts[(size_t)fi * IV_PARTS + part] = o;
    }
}

__global__ void __launch_bounds__(256)
k_inv_finish(const StatsGeom g, const FrameRef* __restrict__ frames, const uint32_t* __restrict__ thr, const InvPart* __restrict__ parts,
             const uint32_t* __restrict__ colpart, int wa, FrameStats* __restrict__ stats, uint32_t* __restrict__ colsum_out,
             int* __restrict__ fail_list, int* __restrict__ fail_count) {
    const int fi = blockIdx.x, tid = threadIdx.x;
    const FrameRef fr = frames[fi];
    if (colsum_out && colpart) {
        const bool aligned = (fr.pitch % 8) == 0;
        const int mis = aligned ? (int)((reinterpret_cast<uintptr_t>(fr.origin) >> 1) & 7) : 0;
        for (int x = tid; x < g.W; x += 256) {
            uint32_t sum = 0;
            for (int p = 0; p < IV_PARTS; p++) sum += colpart[((size_t)fi * IV_PARTS + p) * wa + x + mis];
            colsum_out[(size_t)fi * g.W + x] = sum;
        }
    }
    if (tid != 0) return;
    uint32_t cnt[6] = {0, 0, 0, 0, 0, 0}, mn = 0xffffu, mx = 0;
    unsigned long long total = 0;
    for (int p = 0; p < IV_PARTS; p++) {
        const InvPart& o = parts[(size_t)fi * IV_PARTS + p];
        for (int t = 0; t < 6; t++) cnt[t] += o.cnt[t];
        mn = min(mn, o.mn);
        mx = max(mx, o.mx);
        total += o.total;
    }
    const uint32_t npix = (uint32_t)g.H * (uint32_t)g.W;
    bool ok = true;
    double L[3], U[3];
    for (int q = 0; q < 3; q++) {
        const uint32_t TL = thr[fi * 6 + 2 * q], TU = thr[fi * 6 + 2 * q + 1];
        const uint32_t cL = cnt[2 * q], cU = TU >= 65536u ? npix : cnt[2 * q + 1];
        // #(v < TL) <= rank_prev: the order statistic at rank_prev is >= TL; #(v < TU) >= rank_next + 1: the one at rank_next is < TU
        ok = ok && cL <= g.ranks[2 * q] && cU >= g.ranks[2 * q + 1] + 1u;
        L[q] = (double)TL;
        U[q] = (double)TU - 1.0;
    }
    // |p_mid - p_low| = p_mid - p_low, |p_mid - p_high| = p_high - p_mid (percentiles are monotone in q)
    const double a_lo = fmax(0.0, L[1] - U[0]), a_hi = fmax(0.0, U[1] - L[0]);
    const double b_lo = fmax(0.0, L[2] - U[1]), b_hi = fmax(0.0, U[2] - L[1]);
    int code = 0;
    if (ok && a_lo > b_hi) code = 3;            // certainly inverted
    else if (ok && a_hi < b_lo) code = 2;       // certainly not inverted
    FrameStats& o = stats[fi];
    o.mn = mn;
    o.mx = mx;
    o.npix = npix;
    o.sum = total;
    o.corner_sum = 0;
    o.inv_certified = (uint32_t)code;
    for (int k = 0; k < STATS_MAX_RANKS; k++) o.ostat[k] = 0;
    if (code == 0) fail_list[atomicAdd(fail_count, 1)] = fi;
}

__global__ void k_inv_gather_refs(const FrameRef* __restrict__ frames, const int* __restrict__ list, int m, FrameRef* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) out[i] = frames[list[i]];
}

__global__ void k_inv_scatter_ostat(const FrameStats* __restrict__ src, const int* __restrict__ list, int m, FrameStats* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    FrameStats& d = dst[list[i]];
    for (int k = 0; k < STATS_MAX_RANKS; k++) d.ostat[k] = src[i].ostat[k];
    d.inv_certified = 0;
}

template <int VPL>
static void launch_inv_stream(cudaStream_t st, bool cols, const StatsGeom& g, const FrameRef* refs, int n, const uint32_t* thr, InvPart* parts,
                              uint32_t* rowsum, uint32_t* colpart, int wa) {
    if (cols) k_inv_stream<VPL, true><<<dim3(IV_PARTS, n), IV_THREADS, sizeof(uint32_t) * wa, st>>>(g, refs, thr, parts, rowsum, colpart, wa);
    else k_inv_stream<VPL, false><<<dim3(IV_PARTS, n), IV_THREADS, 0, st>>>(g, refs, thr, parts, rowsum, nullptr, wa);
}

// g.ranks = (prev, next) of the low, middle and high percentile; box must be 0.  Returns with d_stats complete: inv_certified >= 2 carries
// the certified decision (2 + inverted, ostat unused), inv_certified == 0 exact ostat from the histogram path.  One host round trip
// (count of the uncertified frames).
int launch_frame_stats_inversion(epid_ctx* ctx, cudaStream_t stream, const StatsGeom& g, const FrameRef* d_frames, int n, FrameStats* d_stats,
                                 uint32_t* d_rowsum, uint32_t* d_colsum) {
    if (ctx->stats_exact || g.nranks != 6 || g.box > 0 || g.W > 2040 || g.H < IV_SAMPLE_ROWS || g.W < 8)
        return launch_frame_stats(ctx, stream, g, d_frames, n, d_stats, d_rowsum, d_colsum);
    const int nvec = (g.W + 7 + 7) / 8;
    const int vpl = (nvec + 31) / 32;
    const int wa = vpl * 32 * 8;
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    const size_t o_thr = sz(sizeof(uint32_t) * 6 * (size_t)n), o_parts = sz(sizeof(InvPart) * (size_t)n * IV_PARTS);
    const size_t o_list = sz(sizeof(int) * ((size_t)n + 1)), o_refs = sz(sizeof(FrameRef) * (size_t)n), o_tmp = sz(sizeof(FrameStats) * (size_t)n);
    const size_t o_col = sz(d_colsum ? sizeof(uint32_t) * (size_t)n * IV_PARTS * wa : 0);
    if (ctx->inv_bytes < o) {
        if (ctx->inv_scratch) { EPID_CUDA(cudaStreamSynchronize(stream)); EPID_CUDA(cudaFree(ctx->inv_scratch)); ctx->inv_scratch = nullptr; ctx->inv_bytes = 0; }
        cudaError_t e = cudaMalloc(&ctx->inv_scratch, o);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", o, cudaGetErrorString(e)); return EPID_ERR_NOMEM; }
        ctx->inv_bytes = o;
    }
    char* base = (char*)ctx->inv_scratch;
    uint32_t* thr = (uint32_t*)(base + o_thr);
    InvPart* parts = (InvPart*)(base + o_parts);
    int* list = (int*)(base + o_list);       // [0] = count, then the frame indices
    FrameRef* refs2 = (FrameRef*)(base + o_refs);
    FrameStats* tmp = (FrameStats*)(base + o_tmp);
    uint32_t* colpart = d_colsum ? (uint32_t*)(base + o_col) : nullptr;
    EPID_CUDA(cudaMemsetAsync(list, 0, sizeof(int), stream));
    k_inv_pilot<<<n, IV_THREADS, 0, stream>>>(g, d_frames, thr);
    const bool cols = d_colsum != nullptr;
    if (vpl <= 4) launch_inv_stream<4>(stream, cols, g, d_frames, n, thr, parts, d_rowsum, colpart, wa);
    else if (vpl <= 6) launch_inv_stream<6>(stream, cols, g, d_frames, n, thr, parts, d_rowsum, colpart, wa);
    else launch_inv_stream<8>(stream, cols, g, d_frames, n, thr, parts, d_rowsum, colpart, wa);
    k_inv_finish<<<n, 256, 0, stream>>>(g, d_frames, thr, parts, colpart, wa, d_stats, d_colsum, list + 1, list);
    ctx->launches += 3;
    EPID_CUDA(cudaGetLastError());
    int m = 0;
    EPID_CUDA(cudaMemcpyAsync(&m, list, sizeof(int), cudaMemcpyDeviceToHost, stream));
    EPID_CUDA(cudaStreamSynchronize(stream));
    ctx->stats_uncertified += m;
    if (m > 0) {       // exact order statistics for the frames whose decision could not be certified
        k_inv_gather_refs<<<(m + 127) / 128, 128, 0, stream>>>(d_frames, list + 1, m, refs2);
        int rc = launch_frame_stats(ctx, stream, g, refs2, m, tmp, nullptr, nullptr);
        if (rc != EPID_OK) return rc;
        k_inv_scatter_ostat<<<(m + 127) / 128, 128, 0, stream>>>(tmp, list + 1, m, d_stats);
        ctx->launches += 2;
        EPID_CUDA(cudaGetLastError());
    }
    return EPID_OK;
}

}  // namespace epid
