// Single-pass front end of the batched PicketFence pipeline (replaces the two-sweep kernel of round 1a):
//
//   k_pf_pilot   every 32nd row (3 % of the frame): sample-guided thresholds  u_lo, [a1, b1], l_hi  around the ranks of
//                p0.5, the median pair and p99.5
//   k_pf_stream  ONE read of every frame through a TMA (cp.async.bulk) ring: min / max, raw row + column sums, row +
//                column sums of max(v, a1), the exact pixel counts #(v < a1), #(v <= b1) and lower bounds of #(v <= u_lo),
//                #(v >= l_hi) (counts of 4-pixel groups whose minimum / maximum passes the threshold)
//   k_pf_tail    per frame: combine the partial sums, CERTIFY every decision of the reference's front end from the exact
//                counts, then orientation / leaf profile / picket search (pf_profile_block)
//
// Reference semantics: PFDicomImage._has_noise / check_inversion (picketfence.py:221-238, core/image.py:868-897),
// ground + normalize (picketfence.py:322-323), PicketFence.orientation (picketfence.py:1501-1526), picket search
// (picketfence.py:747-767).
//
// Why certification instead of exact order statistics.  The reference uses np.percentile(frame, [0.5, 99.5]) and
// np.median(frame) only inside comparisons:
//   * _has_noise: max > 1.25 * p99.5  or  (min < 0.75 * p0.5 and |min - p0.5| > 0.1 * (p99.5 - p0.5)).  The predicate is
//     monotone (rising in p0.5, falling in p99.5).  #(v <= u_lo) >= rank + 1 proves p0.5 <= u_lo and #(v >= l_hi) >= npix - rank
//     proves p99.5 >= l_hi; if the predicate is false at (u_lo, l_hi) it is false for the true percentiles.
//   * orientation: the median enters as the clamp level of sum(max(pixel, median)) per row / column.  #(v < a1) <= rank and
//     #(v <= b1) >= rank + 1 prove a1 <= median <= b1, every clamped sum then lies within Delta = 2 (b1 - a1) * (pixels per
//     line) of the sum clamped at a1, so does every percentile of the sums, and "row_range < col_range" is decided with
//     that margin.
// A frame whose decisions cannot be certified (noisy frame, nearly square percentile ranges, a pilot band that missed its
// rank) is counted in counters[1] and re-run by the exact histogram pipeline (pf.cu), so results never depend on the
// sample.  Everything downstream (profile, pickets, windows) uses exact integer sums and is bit-identical to that pipeline.
//
// Stream kernel structure (sm_90a): one persistent CTA per SM; a producer warp issues one cp.async.bulk per frame row
// into a ring of stages (mbarrier complete_tx), 12 consumer warps take one row each per stage with conflict-free LDS.128;
// every lane owns up to 4 aligned 8-pixel vectors of the row, so the column sums stay in registers for a whole work item
// (a block of rows of one frame) and are reduced across warps through shared memory once per item.  All per-pixel work is
// packed u16x2 arithmetic (VIMNMX.U16x2, IDP.2A), branch free: ~12 integer instructions per pixel.
// PicketFence profiles have ~1000 samples: find_peaks' 32-sample skip table (peaks.cuh) buys nothing here, and its 9 KB of static shared
// memory cost k_pf_tail a resident CTA per SM
#define EPID_PK_MAXBLK 2
#include "pf_common.cuh"
#include "tma.cuh"

namespace epid {

// ------------------------------------------------------------------------------------------------ shared definitions
#ifndef EPID_ST_NCW
#define EPID_ST_NCW 12
#endif
constexpr int ST_NCW = EPID_ST_NCW;                 // consumer warps
constexpr int ST_THREADS = (ST_NCW + 1) * 32;
constexpr int ST_NST = 6;                  // ring stages
constexpr int ST_KMAX = 8;                 // max row blocks (items) per frame
constexpr int ST_MAXROWS = 1024;           // rows per item
constexpr int PILOT_THREADS = 256;
constexpr int PILOT_BINS = 2048;
constexpr int PILOT_STEP = 32, PILOT_OFF = 16;
constexpr int TAIL_THREADS = 256;

struct PilotOut {            // thresholds of one frame (raw pixel values)
    uint32_t u_lo, a1, b1, l_hi;
};

struct ItemOut {             // per work item (row block of a frame)
    uint32_t mn, mx;
    uint32_t cnt_a, cnt_b, cnt_lo, cnt_hi;
    uint32_t pad[2];
};

struct StreamGeom {
    int H, W;
    int K;                   // items per frame
    int rows_per_item;
    int nvec;                // vectors of the aligned 8-pixel grid that cover one row of the view
    int nstrips;             // 1 or 2 column strips (a consumer warp owns one strip)
    int wa;                  // aligned columns per item in the partial-sum arrays = nstrips * VPL * 256
    int row_bytes;           // nvec * 16
    int rps;                 // rows per stage = ST_NCW / nstrips
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(ST_NCW * 32) : "memory"); }
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}

__device__ __forceinline__ int pilot_rows_of(int H) { return H > PILOT_OFF ? (H - PILOT_OFF + PILOT_STEP - 1) / PILOT_STEP : 0; }

// ------------------------------------------------------------------------------------------------ pilot
// exclusive block scan over PILOT_THREADS threads; returns the exclusive prefix, *total = block sum
__device__ __forceinline__ uint32_t pilot_scan_excl(uint32_t v, uint32_t* s_red, uint32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) s_red[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const uint32_t w = lane < PILOT_THREADS / 32 ? s_red[lane] : 0;
        uint32_t winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += t;
        }
        if (lane < PILOT_THREADS / 32) s_red[lane] = winc - w;
        if (lane == 31) s_red[32] = winc;
    }
    __syncthreads();
    const uint32_t excl = s_red[wid] + inc - v;
    *total = s_red[32];
    return excl;
}

// smallest bin x in [0, nb) with base + sum(hist[0..x]) > rank; nb if the band ends first, 0xffffffff if rank < base
__device__ inline uint32_t pilot_find(const uint32_t* __restrict__ hist, uint32_t nb, uint32_t base, uint32_t rank, uint32_t* s_red,
                                      uint32_t* s_found) {
    const int tid = threadIdx.x;
    const uint32_t per = (nb + PILOT_THREADS - 1) / PILOT_THREADS;
    const uint32_t lo = min(nb, tid * per), hi = min(nb, lo + per);
    uint32_t c = 0;
    for (uint32_t i = lo; i < hi; i++) c += hist[i];
    uint32_t total;
    const uint32_t excl = pilot_scan_excl(c, s_red, &total);
    if (tid == 0) *s_found = rank < base ? 0xffffffffu : nb;
    __syncthreads();
    if (rank >= base) {
        const uint32_t k = rank - base;
        if (k >= excl && k < excl + c) {
            uint32_t acc = excl;
            for (uint32_t i = lo; i < hi; i++) {
                const uint32_t h = hist[i];
                if (k < acc + h) { *s_found = i; break; }
                acc += h;
            }
        }
    }
    __syncthreads();
    const uint32_t r = *s_found;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(PILOT_THREADS)
k_pf_pilot(const StatsGeom g, const FrameRef* __restrict__ frames, int nframes, PilotOut* __restrict__ out) {
    __shared__ uint32_t hist[3][PILOT_BINS];
    __shared__ uint32_t bis_lo[4], bis_hi[4], bis_cnt[4], bis_rank[4];
    __shared__ uint32_t a0s[3], b0s[3], shs[3], below_s[3], eq_s[3];
    __shared__ uint32_t s_red[40], s_found, smin, smax;
    const int fi = blockIdx.x;
    if (fi >= nframes) return;
    const FrameRef frf = frames[fi];
    const int H = g.H, W = g.W;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t npix = (uint32_t)H * (uint32_t)W;
    // ranks (band domain): lo pair (raw), median pair (raw), hi pair (flipped: v' = 65535 - v)
    const uint32_t k_lo[3] = {g.ranks[0], g.ranks[4], npix - 1 - g.ranks[3]};
    const uint32_t k_hi[3] = {g.ranks[1], g.ranks[5], npix - 1 - g.ranks[2]};
    for (int i = tid; i < 3 * PILOT_BINS; i += PILOT_THREADS) (&hist[0][0])[i] = 0;
    if (tid < 3) { below_s[tid] = 0; eq_s[tid] = 0; }
    if (tid == 0) { smin = 0xffffu; smax = 0; }
    // ---- T0: 2048-pixel grid sample (8 rows x 256 columns), 16-step value bisection -> wide bands
    uint32_t sv[8];
    {
        const int col = min(W - 1, (int)(((long long)tid * W) / PILOT_THREADS));
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int row = min(H - 1, (int)(((2 * i + 1) * (long long)H) / 16));
            sv[i] = __ldg(frf.origin + (size_t)row * frf.pitch + col);
        }
    }
    const uint32_t nT0 = PILOT_THREADS * 8;
    if (tid < 4) {
        // t0: band 0 upper, t1: band 1 lower, t2: band 1 upper, t3: band 2 upper (flipped); margins 5 sigma
        const int b = tid == 0 ? 0 : (tid == 3 ? 2 : 1);
        // bands 0 / 2 are taken on the minima / maxima of 4-pixel groups: the rank sits at a 4x higher quantile there
        const double fq = fmin((b == 1 ? 1.0 : 4.0) * (double)(tid == 1 ? k_lo[b] : k_hi[b]) / (double)npix, 0.999);
        const double sg = sqrt(fq * (1.0 - fq) * (double)nT0);
        const double ctr = fq * (double)nT0;
        double rr = (tid == 1) ? ctr - 5.0 * sg - 2.0 : ctr + 5.0 * sg + 3.0;
        rr = fmin(fmax(rr, 0.0), (double)(nT0 - 1));
        bis_rank[tid] = (uint32_t)rr;
        bis_lo[tid] = 0;
        bis_hi[tid] = 65535u;
        bis_cnt[tid] = 0;
    }
    __syncthreads();
    {
        uint32_t mnv = sv[0], mxv = sv[0];
#pragma unroll
        for (int i = 1; i < 8; i++) { mnv = min(mnv, sv[i]); mxv = max(mxv, sv[i]); }
        mnv = warp_min(mnv);
        mxv = warp_max(mxv);
        if (lane == 0) { atomicMin(&smin, mnv); atomicMax(&smax, mxv); }
    }
    for (int step = 0; step < 16; step++) {
        uint32_t cnt[4];
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const uint32_t mid = (bis_lo[t] + bis_hi[t]) >> 1;
            uint32_t cc_ = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t v = t == 3 ? 65535u - sv[i] : sv[i];
                cc_ += v <= mid ? 1u : 0u;
            }
            cnt[t] = __reduce_add_sync(0xffffffffu, cc_);
        }
        if (lane < 4) atomicAdd(&bis_cnt[lane], lane == 0 ? cnt[0] : lane == 1 ? cnt[1] : lane == 2 ? cnt[2] : cnt[3]);
        __syncthreads();
        if (tid < 4) {
            const uint32_t mid = (bis_lo[tid] + bis_hi[tid]) >> 1;
            if (bis_cnt[tid] >= bis_rank[tid] + 1) bis_hi[tid] = mid; else bis_lo[tid] = mid + 1;
            bis_cnt[tid] = 0;
        }
        __syncthreads();
    }
    if (tid == 0) {
        // band 0: [sample min, q(upper)], band 1: [q(lower), q(upper)], band 2 (flipped): [65535 - sample max, q'(upper)];
        // bins of 2^sh values so that any band fits the histogram (the thresholds only need that granularity)
        uint32_t a[3], b[3];
        a[0] = smin;              b[0] = max(bis_lo[0], smin);
        a[1] = bis_lo[1];         b[1] = max(bis_lo[2], a[1]);
        a[2] = 65535u - smax;     b[2] = max(bis_lo[3], a[2]);
        for (int j = 0; j < 3; j++) {
            uint32_t sh = 0;
            while (((b[j] - a[j]) >> sh) >= (uint32_t)PILOT_BINS) sh++;
            a0s[j] = a[j];
            b0s[j] = b[j];
            shs[j] = sh;
        }
    }
    __syncthreads();
    // ---- pilot rows: pixels below a band are counted in registers, pixels equal to its lower edge too (heavy ties such
    // as a clipped floor), pixels inside go to the band histogram
    const uint32_t a0[3] = {a0s[0], a0s[1], a0s[2]};
    const uint32_t wd[3] = {b0s[0] - a0s[0], b0s[1] - a0s[1], b0s[2] - a0s[2]};
    const uint32_t sh[3] = {shs[0], shs[1], shs[2]};
    uint32_t below[3] = {0, 0, 0}, eq[3] = {0, 0, 0};
    const int np_rows = pilot_rows_of(H);
    const bool aligned = true;    // pf_front_supported(): pitch % 8 == 0
    const int mis = (int)((reinterpret_cast<uintptr_t>(frf.origin) >> 1) & 7);
    const int jf = (mis + 7) / 8, jl = (W + mis) / 8;                       // full vectors [jf, jl) cover view columns [cl, cr)
    const int cl = aligned ? min(W, max(0, jf * 8 - mis)) : 0;
    const int cr = aligned ? (jl > jf ? jl * 8 - mis : cl) : 0;
    // band 1 (median): every pixel; bands 0 / 2 (extremes): the minimum / maximum of each group of 4 alternate pixels of an
    // aligned vector -- the statistic whose count the stream kernel certifies (#groups with min <= u_lo is a lower bound of
    // #pixels <= u_lo)
    auto put = [&](int j, uint32_t vv) {
        const int u = (int)vv - (int)a0[j];
        below[j] += (uint32_t)u >> 31;
        eq[j] += u == 0 ? 1u : 0u;
        if ((uint32_t)(u - 1) < wd[j]) atomicAdd(&hist[j][(uint32_t)u >> sh[j]], 1u);
    };
    for (int ri = wid; ri < np_rows; ri += PILOT_THREADS / 32) {
        const uint16_t* rowp = frf.origin + (size_t)(PILOT_OFF + PILOT_STEP * ri) * frf.pitch;
        for (int j = jf + lane; j < jl; j += 32) {
            const uint4 q = ldg_stream16(rowp - mis + j * 8);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
            const uint32_t vm = __vminu2(__vminu2(w[0], w[1]), __vminu2(w[2], w[3]));
            const uint32_t vM = __vmaxu2(__vmaxu2(w[0], w[1]), __vmaxu2(w[2], w[3]));
            put(0, vm & 0xffffu);
            put(0, vm >> 16);
            put(2, 65535u - (vM & 0xffffu));
            put(2, 65535u - (vM >> 16));
#pragma unroll
            for (int t = 0; t < 4; t++) { put(1, w[t] & 0xffffu); put(1, w[t] >> 16); }
        }
    }
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const uint32_t b = __reduce_add_sync(0xffffffffu, below[j]);
        const uint32_t e = __reduce_add_sync(0xffffffffu, eq[j]);
        if (lane == 0) { if (b) atomicAdd(&below_s[j], b); if (e) atomicAdd(&eq_s[j], e); }
    }
    __syncthreads();
    if (tid < 3 && eq_s[tid]) hist[tid][0] += eq_s[tid];
    __syncthreads();
    // ---- thresholds from the pilot histograms (ranks scaled to the pilot subset, +-5 sigma)
    const uint32_t n_p = (uint32_t)np_rows * (uint32_t)(aligned ? cr - cl : W);
    uint32_t thr_lo[3], thr_hi[3];      // band domain: lower-edge threshold for k_lo, upper-edge threshold for k_hi
    for (int j = 0; j < 3; j++) {
        const uint32_t nb = (wd[j] >> sh[j]) + 1;
        // population of the pilot statistic: pixels (band 1) or 4-pixel groups (bands 0 / 2); an absolute full-frame count k
        // is expected at k * n_p / npix in either population
        const double scale = (double)n_p / (double)npix;
        const double pop = j == 1 ? (double)n_p : (double)n_p / 4.0;
        const double fq = fmin((j == 1 ? 1.0 : 4.0) * ((double)k_lo[j] + 0.5) / (double)npix, 1.0);
        const double sg = sqrt(fq * (1.0 - fq) * pop);
        const double rl = (double)k_lo[j] * scale - 5.0 * sg - 2.0;
        const double ru = (double)k_hi[j] * scale + 5.0 * sg + 3.0;
        const uint32_t r_l = rl <= 0.0 ? 0u : (uint32_t)rl;
        const uint32_t r_u = (uint32_t)fmin(ru, fmax(pop - 1.0, 0.0));
        const uint32_t xa = pilot_find(hist[j], nb, below_s[j], r_l, s_red, &s_found);
        const uint32_t xb = pilot_find(hist[j], nb, below_s[j], r_u, s_red, &s_found);
        // lower threshold: lower edge of bin xa (rank below the band: the band's lower edge; beyond: its upper edge)
        uint32_t lo_t = xa == 0xffffffffu ? a0[j] : a0[j] + (min(xa, nb - 1) << sh[j]);
        // upper threshold: upper edge of bin xb (clamped to the band / 16 bit)
        uint32_t hi_t = xb == 0xffffffffu ? a0[j] : a0[j] + (((min(xb, nb - 1) + 1) << sh[j]) - 1);
        hi_t = min(hi_t, 65535u);
        lo_t = min(lo_t, hi_t);
        thr_lo[j] = lo_t;
        thr_hi[j] = hi_t;
    }
    if (tid == 0) {
        PilotOut o;
        o.u_lo = thr_hi[0];
        o.a1 = thr_lo[1];
        o.b1 = thr_hi[1];
        o.l_hi = 65535u - thr_hi[2];
        out[fi] = o;
    }
}

// ------------------------------------------------------------------------------------------------ stream
struct StreamSh {
    unsigned long long full[ST_NST], empty[ST_NST];
    uint32_t mn, mx, cnt[4];
};

template <int VPL>
__global__ void __launch_bounds__(ST_THREADS, 1)
k_pf_stream(const StreamGeom sg, const FrameRef* __restrict__ frames, const PilotOut* __restrict__ pilot, int nitems,
            ItemOut* __restrict__ items, uint32_t* __restrict__ col_raw, uint32_t* __restrict__ col_cl,
            uint32_t* __restrict__ row_raw, uint32_t* __restrict__ row_cl) {
    extern __shared__ __align__(128) unsigned char smraw[];
    StreamSh* sh = reinterpret_cast<StreamSh*>(smraw);
    unsigned char* ring = smraw + 256;
    const int stage_bytes = sg.rps * sg.row_bytes;
    uint32_t* flush = reinterpret_cast<uint32_t*>(ring + (size_t)ST_NST * stage_bytes);   // [ST_NCW][VPL * 256]
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < ST_NST; s++) { mbar_init(smem_u32(&sh->full[s]), 1); mbar_init(smem_u32(&sh->empty[s]), ST_NCW); }
        sh->mn = 0xffffu;
        sh->mx = 0;
        sh->cnt[0] = sh->cnt[1] = sh->cnt[2] = sh->cnt[3] = 0;
        mbar_fence_init();
    }
    __syncthreads();
    const int H = sg.H, W = sg.W;
    if (wid == ST_NCW) {
        // ================= producer: one cp.async.bulk per frame row, lanes issue the rows of a stage in parallel
        int st = 0;
        uint32_t ph = 0;
        for (int it = blockIdx.x; it < nitems; it += gridDim.x) {
            const int fi = it / sg.K, blk = it - fi * sg.K;
            const FrameRef frf = frames[fi];
            const int mis = (int)((reinterpret_cast<uintptr_t>(frf.origin) >> 1) & 7);
            const uint16_t* base = frf.origin - mis;
            const uint32_t bytes = (uint32_t)((W + mis + 7) / 8) * 16u;   // aligned-grid vectors that cover this frame's rows
            const int r0 = blk * sg.rows_per_item, r1 = min(H, r0 + sg.rows_per_item);
            for (int rr = r0; rr < r1; rr += sg.rps) {
                const int nrows = min(sg.rps, r1 - rr);
                mbar_wait(smem_u32(&sh->empty[st]), ph ^ 1u);
                if (lane == 0) mbar_expect_tx(smem_u32(&sh->full[st]), (uint32_t)nrows * bytes);
                __syncwarp();
                if (lane < nrows)
                    tma_load_1d(smem_u32(ring + (size_t)st * stage_bytes + (size_t)lane * sg.row_bytes),
                                base + (size_t)(rr + lane) * frf.pitch, bytes, smem_u32(&sh->full[st]));
                if (++st == ST_NST) { st = 0; ph ^= 1u; }
            }
        }
        return;
    }
    // ================= consumers
    const int strip = wid % sg.nstrips, rslot = wid / sg.nstrips;
    const int ctid = tid;                                  // consumer thread index (warps 0 .. ST_NCW-1)
    uint32_t cs_raw[VPL * 8], cs_cl[VPL * 8];
#pragma unroll
    for (int i = 0; i < VPL * 8; i++) { cs_raw[i] = 0; cs_cl[i] = 0; }
    int st = 0;
    uint32_t ph = 0;
    for (int it = blockIdx.x; it < nitems; it += gridDim.x) {
        const int fi = it / sg.K, blk = it - fi * sg.K;
        const FrameRef frf = frames[fi];
        const int mis = (int)((reinterpret_cast<uintptr_t>(frf.origin) >> 1) & 7);
        const PilotOut po = pilot[fi];
        const int r0 = blk * sg.rows_per_item, r1 = min(H, r0 + sg.rows_per_item);
        // packed thresholds: [v < a1], [v <= b1] = [v < b1 + 1], [v <= u_lo] = [v < u_lo + 1], [v >= l_hi] = [v > l_hi - 1]
        const uint32_t Ap = po.a1 * 0x00010001u;
        const uint32_t Bp = min(po.b1 + 1u, 65535u) * 0x00010001u;
        const uint32_t Up = min(po.u_lo + 1u, 65535u) * 0x00010001u;
        const uint32_t Lp = (po.l_hi > 0 ? po.l_hi - 1u : 0u) * 0x00010001u;
        bool full[VPL];
        uint32_t voff[VPL];
#pragma unroll
        for (int v = 0; v < VPL; v++) {
            const int j = strip * VPL * 32 + lane + 32 * v;
            const int c0 = j * 8 - mis;
            full[v] = j < sg.nvec && c0 >= 0 && c0 + 8 <= W;
            voff[v] = (uint32_t)j * 16u;
        }
        uint32_t mn2 = 0xffffffffu, mx2 = 0, cA = 0, cB = 0, cL = 0, cH = 0;
        for (int rr = r0; rr < r1; rr += sg.rps) {
            mbar_wait(smem_u32(&sh->full[st]), ph);
            const int row = rr + rslot;
            if (row < r1) {
                const uint32_t rbase = smem_u32(ring + (size_t)st * stage_bytes + (size_t)rslot * sg.row_bytes);
                uint4 q[VPL];
#pragma unroll
                for (int v = 0; v < VPL; v++) q[v] = full[v] ? lds128(rbase + voff[v]) : make_uint4(0, 0, 0, 0);
                uint32_t rs = 0, rc = 0;
#pragma unroll
                for (int v = 0; v < VPL; v++) {
                    if (full[v]) {
                        const uint32_t w[4] = {q[v].x, q[v].y, q[v].z, q[v].w};
                        // packed min / max of the vector: each half = a group of 4 alternate pixels
                        const uint32_t vm = __vminu2(__vminu2(w[0], w[1]), __vminu2(w[2], w[3]));
                        const uint32_t vM = __vmaxu2(__vmaxu2(w[0], w[1]), __vmaxu2(w[2], w[3]));
                        mn2 = __vminu2(mn2, vm);
                        mx2 = __vmaxu2(mx2, vM);
                        // groups whose minimum is <= u_lo / whose maximum is >= l_hi: lower bounds of the pixel counts
                        cL = __dp2a_lo(__vminu2(__vmaxu2(vm, Up) - vm, 0x00010001u), 0x0101u, cL);
                        cH = __dp2a_lo(__vminu2(vM - __vminu2(vM, Lp), 0x00010001u), 0x0101u, cH);
#pragma unroll
                        for (int t = 0; t < 4; t++) {
                            const uint32_t x = w[t];
                            cs_raw[v * 8 + 2 * t] = __dp2a_lo(x, 0x0001u, cs_raw[v * 8 + 2 * t]);
                            cs_raw[v * 8 + 2 * t + 1] = __dp2a_lo(x, 0x0100u, cs_raw[v * 8 + 2 * t + 1]);
                            rs = __dp2a_lo(x, 0x0101u, rs);
                            const uint32_t xa = __vmaxu2(x, Ap);
                            cs_cl[v * 8 + 2 * t] = __dp2a_lo(xa, 0x0001u, cs_cl[v * 8 + 2 * t]);
                            cs_cl[v * 8 + 2 * t + 1] = __dp2a_lo(xa, 0x0100u, cs_cl[v * 8 + 2 * t + 1]);
                            rc = __dp2a_lo(xa, 0x0101u, rc);
                            cA = __dp2a_lo(__vminu2(xa - x, 0x00010001u), 0x0101u, cA);
                            cB = __dp2a_lo(__vminu2(__vmaxu2(x, Bp) - x, 0x00010001u), 0x0101u, cB);
                        }
                    }
                }
                rs = __reduce_add_sync(0xffffffffu, rs);
                rc = __reduce_add_sync(0xffffffffu, rc);
                if (lane == 0) {
                    row_raw[((size_t)fi * 2 + strip) * H + row] = rs;
                    row_cl[((size_t)fi * 2 + strip) * H + row] = rc;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&sh->empty[st]));
            if (++st == ST_NST) { st = 0; ph ^= 1u; }
        }
        // ---- item end: scalars through shared atomics, column sums through the flush buffer
        {
            uint32_t mnv = min(mn2 & 0xffffu, mn2 >> 16), mxv = max(mx2 & 0xffffu, mx2 >> 16);
            mnv = __reduce_min_sync(0xffffffffu, mnv);
            mxv = __reduce_max_sync(0xffffffffu, mxv);
            cA = __reduce_add_sync(0xffffffffu, cA);
            cB = __reduce_add_sync(0xffffffffu, cB);
            cL = __reduce_add_sync(0xffffffffu, cL);
            cH = __reduce_add_sync(0xffffffffu, cH);
            if (lane == 0) {
                atomicMin(&sh->mn, mnv);
                atomicMax(&sh->mx, mxv);
                atomicAdd(&sh->cnt[0], cA);
                atomicAdd(&sh->cnt[1], cB);
                atomicAdd(&sh->cnt[2], cL);
                atomicAdd(&sh->cnt[3], cH);
            }
        }
        uint32_t* mine = flush + (size_t)wid * (VPL * 256);
        const int group = ST_NCW / sg.nstrips;               // warps per strip
#pragma unroll
        for (int arr = 0; arr < 2; arr++) {
#pragma unroll
            for (int kp = 0; kp < VPL * 8; kp++) mine[kp * 32 + lane] = arr == 0 ? cs_raw[kp] : cs_cl[kp];
            consumer_bar();
            if (arr == 0 && ctid == 0) {
                ItemOut o;
                o.mn = sh->mn; o.mx = sh->mx;
                o.cnt_a = sh->cnt[0]; o.cnt_b = sh->cnt[1]; o.cnt_lo = sh->cnt[2]; o.cnt_hi = sh->cnt[3];
                o.pad[0] = o.pad[1] = 0;
                items[it] = o;
                sh->mn = 0xffffu; sh->mx = 0;
                sh->cnt[0] = sh->cnt[1] = sh->cnt[2] = sh->cnt[3] = 0;
            }
            uint32_t* dst = (arr == 0 ? col_raw : col_cl) + (size_t)it * sg.wa;
            for (int idx = ctid; idx < sg.nstrips * VPL * 256; idx += ST_NCW * 32) {
                const int sp = idx / (VPL * 256), loc = idx - sp * (VPL * 256);
                uint32_t s = 0;
                for (int k = 0; k < group; k++) s += flush[(size_t)(k * sg.nstrips + sp) * (VPL * 256) + loc];
                const int kp = loc >> 5, ln = loc & 31;
                const int v = kp >> 3, p = kp & 7;
                const int j = sp * VPL * 32 + ln + 32 * v;
                dst[j * 8 + p] = s;
            }
            consumer_bar();
        }
#pragma unroll
        for (int i = 0; i < VPL * 8; i++) { cs_raw[i] = 0; cs_cl[i] = 0; }
    }
}

// ------------------------------------------------------------------------------------------------ tail
// 4 CTAs / SM: 512 frames fit in one wave of an H100's 132 SMs (the kernel is a chain of short block-wide phases: latency, not issue)
__global__ void __launch_bounds__(TAIL_THREADS, 4)
k_pf_tail(const PfConst* __restrict__ cc, const StatsGeom g, const StreamGeom sg, const FrameRef* __restrict__ frames,
          const PilotOut* __restrict__ pilot, const ItemOut* __restrict__ items, const uint32_t* __restrict__ col_raw,
          const uint32_t* __restrict__ col_cl, const uint32_t* __restrict__ row_raw, const uint32_t* __restrict__ row_cl,
          PfFrame* fr, FrameStats* __restrict__ stats, int* counters) {
    extern __shared__ __align__(128) unsigned char smraw[];
    __shared__ uint32_t s_mn, s_mx, s_cnt[4], s_flag;
    __shared__ unsigned long long s_sum, s_corner;
    const PfConst& c = *cc;
    const int fi = blockIdx.x;
    const int H = g.H, W = g.W;
    const int Hp = (H + 3) & ~3, Wp = (W + 3) & ~3;
    uint32_t* rowsum_sm = reinterpret_cast<uint32_t*>(smraw);
    uint32_t* colsum_sm = rowsum_sm + Hp;
    uint32_t* rowsum2_sm = colsum_sm + Wp;
    uint32_t* colsum2_sm = rowsum2_sm + Hp;
    unsigned char* prof_raw = reinterpret_cast<unsigned char*>(colsum2_sm + Wp);
    const int tid = threadIdx.x, lane = tid & 31;
    PfFrame& f = fr[fi];
    const FrameRef frf = frames[fi];
    const PilotOut po = pilot[fi];
    const int mis = (int)((reinterpret_cast<uintptr_t>(frf.origin) >> 1) & 7);
    const uint32_t npix = (uint32_t)H * (uint32_t)W;
    if (tid == 0) { s_mn = 0xffffu; s_mx = 0; s_cnt[0] = s_cnt[1] = s_cnt[2] = s_cnt[3] = 0; s_sum = 0; s_corner = 0; s_flag = 0; }
    // ---- combine the partial sums of the frame's items / strips (columns outside the full-vector range stay 0)
    for (int x = tid; x < W; x += TAIL_THREADS) {
        const int ac = x + mis;
        uint32_t a = 0, b = 0;
        if (ac < sg.wa) {
            for (int k = 0; k < sg.K; k++) {
                a += col_raw[((size_t)fi * sg.K + k) * sg.wa + ac];
                b += col_cl[((size_t)fi * sg.K + k) * sg.wa + ac];
            }
        }
        colsum_sm[x] = a;
        colsum2_sm[x] = b;
    }
    for (int y = tid; y < H; y += TAIL_THREADS) {
        uint32_t a = 0, b = 0;
        for (int s = 0; s < sg.nstrips; s++) {
            a += row_raw[((size_t)fi * 2 + s) * H + y];
            b += row_cl[((size_t)fi * 2 + s) * H + y];
        }
        rowsum_sm[y] = a;
        rowsum2_sm[y] = b;
    }
    __syncthreads();
    if (tid < sg.K) {
        const ItemOut o = items[(size_t)fi * sg.K + tid];
        atomicMin(&s_mn, o.mn);
        atomicMax(&s_mx, o.mx);
        atomicAdd(&s_cnt[0], o.cnt_a);
        atomicAdd(&s_cnt[1], o.cnt_b);
        atomicAdd(&s_cnt[2], o.cnt_lo);
        atomicAdd(&s_cnt[3], o.cnt_hi);
    }
    // ---- columns of a misaligned view that no full vector covers (< 8 on each side): scalar pass
    {
        const int jf = (mis + 7) / 8, jl = (W + mis) / 8;
        const int cl = min(W, max(0, jf * 8 - mis)), cr = jl > jf ? jl * 8 - mis : cl;
        const int ne = cl + (W - cr);
        uint32_t mnv = 0xffffu, mxv = 0, e0 = 0, e1 = 0, e2 = 0, e3 = 0;
        for (int i = tid; i < ne * H; i += TAIL_THREADS) {
            const int r = i / ne, e = i - r * ne;
            const int cidx = e < cl ? e : cr + (e - cl);
            const uint32_t v = __ldg(frf.origin + (size_t)r * frf.pitch + cidx);
            const uint32_t xa = max(v, po.a1);
            mnv = min(mnv, v);
            mxv = max(mxv, v);
            atomicAdd(&rowsum_sm[r], v);
            atomicAdd(&colsum_sm[cidx], v);
            atomicAdd(&rowsum2_sm[r], xa);
            atomicAdd(&colsum2_sm[cidx], xa);
            e0 += v < po.a1 ? 1u : 0u;
            e1 += v <= po.b1 ? 1u : 0u;
            e2 += v <= po.u_lo ? 1u : 0u;
            e3 += v >= po.l_hi ? 1u : 0u;
        }
        if (ne > 0) {
            mnv = warp_min(mnv); mxv = warp_max(mxv);
            e0 = warp_sum(e0); e1 = warp_sum(e1); e2 = warp_sum(e2); e3 = warp_sum(e3);
            if (lane == 0) {
                atomicMin(&s_mn, mnv); atomicMax(&s_mx, mxv);
                atomicAdd(&s_cnt[0], e0); atomicAdd(&s_cnt[1], e1); atomicAdd(&s_cnt[2], e2); atomicAdd(&s_cnt[3], e3);
            }
        }
    }
    // corner boxes (core/image.py:881-894)
    if (g.box > 0) {
        const int per = g.box * g.box;
        unsigned long long cs = 0;
        for (int i = tid; i < 4 * per; i += TAIL_THREADS) {
            const int b = i / per, o = i - b * per;
            const int y = o / g.box, x = o - y * g.box;
            const int rr = ((b & 2) ? H - g.rp - g.box : g.rp) + y;
            const int cl = ((b & 1) ? W - g.cp - g.box : g.cp) + x;
            if (rr >= 0 && rr < H && cl >= 0 && cl < W) cs += __ldg(frf.origin + (size_t)rr * frf.pitch + cl);
        }
        cs = warp_sum(cs);
        if (lane == 0 && cs) atomicAdd(&s_corner, cs);
    }
    __syncthreads();
    {
        unsigned long long tsum = 0;
        for (int i = tid; i < H; i += TAIL_THREADS) tsum += rowsum_sm[i];
        tsum = warp_sum(tsum);
        if (lane == 0) atomicAdd(&s_sum, tsum);
    }
    __syncthreads();
    // ---- decisions (thread 0): ground / normalise constants, corner inversion, certified "no noise", clamp level
    if (tid == 0) {
        const uint32_t mn = s_mn, mx = s_mx;
        f.status = EPID_PF_OK;
        f.noisy = 0;
        f.noise_passes = 0;
        f.n_pickets = 0;
        f.n_inview = 0;
        f.todo = 0;
        f.win2 = 0;
        f.orientation = 0;
        f.mn = mn;
        f.mx = mx;
        f.D = mx - mn;
        int bad = 0;
        if (f.D == 0) {
            f.status = EPID_PF_FLAT_IMAGE;
            f.inv = 0;
            f.corner_inverted = 0;
            f.med2 = 0;
        } else {
            // check_inversion(box_size=10, position=(0.01, 0.01)) (core/image.py:881-897): exact
            const double avg = (double)s_corner / (double)(4 * 10 * 10);
            const double mean = (double)s_sum / (double)npix;
            f.corner_inverted = avg > mean ? 1 : 0;
            f.inv = f.corner_inverted ^ (c.p.invert ? 1 : 0);
            // exact counts (a threshold of 65535 / 0 makes the packed test of the stream kernel vacuous)
            const uint32_t cnt_a = s_cnt[0];
            const uint32_t cnt_b = po.b1 >= 65535u ? npix : s_cnt[1];
            const uint32_t cnt_lo = po.u_lo >= 65535u ? npix : s_cnt[2];
            const uint32_t cnt_hi = po.l_hi == 0u ? npix : s_cnt[3];
            // median pair within [a1, b1]
            if (!(cnt_a <= g.ranks[4] && cnt_b >= g.ranks[5] + 1u)) bad = 1;
            // _has_noise (picketfence.py:229-238) at the certified corner p0.5 <= u_lo, p99.5 >= l_hi
            if (!(cnt_lo >= g.ranks[1] + 1u && cnt_hi >= npix - g.ranks[2])) bad = 1;
            const double near_min = (double)min(po.u_lo, mx), near_max = (double)max(po.l_hi, mn);
            const double mnv = (double)mn, mxv = (double)mx;
            const bool max_is_extreme = mxv > near_max * 1.25;
            const bool min_is_extreme = (mnv < near_min * 0.75) && (fabs(mnv - near_min) > 0.1 * (near_max - near_min));
            if (max_is_extreme || min_is_extreme) bad = 1;
            f.med2 = f.inv ? 2u * (mx - min(po.a1, mx)) : 2u * (max(po.a1, mn) - mn);
        }
        FrameStats st;
        st.mn = mn; st.mx = mx; st.npix = npix; st.inv_certified = 0;
        st.sum = s_sum; st.corner_sum = s_corner;
        for (int i = 0; i < STATS_MAX_RANKS; i++) st.ostat[i] = 0;
        st.ostat[0] = mn; st.ostat[1] = po.u_lo; st.ostat[2] = po.l_hi; st.ostat[3] = mx; st.ostat[4] = po.a1; st.ostat[5] = po.b1;
        stats[fi] = st;
        if (bad) { atomicAdd(&counters[1], 1); s_flag = 1; f.status = PF_STATUS_DEFERRED; }
    }
    __syncthreads();
    if (s_flag || f.status != EPID_PF_OK) return;
    // ---- clamped sums at the certified lower clamp level a1, in 2g units (picketfence.py:1509-1514)
    double d_row = 0.0, d_col = 0.0;
    if (c.p.orientation < 0) {
        const uint32_t mn = f.mn, mx = f.mx, a1 = po.a1;
        const int inv = f.inv;
        for (int y = tid; y < H; y += TAIL_THREADS) {
            const uint32_t raw = rowsum_sm[y], cl = rowsum2_sm[y];
            rowsum2_sm[y] = !inv ? 2u * cl - 2u * mn * (uint32_t)W : 2u * mx * (uint32_t)W - 2u * (raw + a1 * (uint32_t)W - cl);
        }
        for (int x = tid; x < W; x += TAIL_THREADS) {
            const uint32_t raw = colsum_sm[x], cl = colsum2_sm[x];
            colsum2_sm[x] = !inv ? 2u * cl - 2u * mn * (uint32_t)H : 2u * mx * (uint32_t)H - 2u * (raw + a1 * (uint32_t)H - cl);
        }
        d_row = 2.0 * (double)(po.b1 - po.a1) * (double)W;     // np.sum(temp, 1): every element sums W pixels
        d_col = 2.0 * (double)(po.b1 - po.a1) * (double)H;     // np.sum(temp, 0)
    }
    __syncthreads();
    pf_profile_block(c, f, rowsum_sm, colsum_sm, rowsum2_sm, colsum2_sm, prof_raw, d_col, d_row, counters);
}

// ------------------------------------------------------------------------------------------------ host side
size_t pf_tail_smem_bytes(int H, int W) {
    const int Hp = (H + 3) & ~3, Wp = (W + 3) & ~3;
    return sizeof(uint32_t) * (size_t)(2 * Hp + 2 * Wp) + pf_profile_smem_bytes(TAIL_THREADS, H, W) + 64;
}

static int stream_vpl(int nvec, int* nstrips) {
    int ns = nvec <= 128 ? 1 : 2;
    int vpl = (nvec + 32 * ns - 1) / (32 * ns);
    *nstrips = ns;
    return vpl;
}

bool pf_front_supported(int H, int W, int pitch) {
    if ((pitch % 8) != 0 || H < 64 || W < 64 || H > STATS_MAX_DIM || W > STATS_MAX_DIM) return false;
    int ns;
    const int nvec = (W + 7 + 7) / 8;
    const int vpl = stream_vpl(nvec, &ns);
    if (vpl > 4) return false;
    if ((H + ST_KMAX - 1) / ST_KMAX > ST_MAXROWS) return false;
    return pf_tail_smem_bytes(H, W) <= 200 * 1024;
}

size_t pf_front_scratch_bytes(int n, int H, int W) {
    // pilot + items + column partials (ST_KMAX items per frame, up to 2048 aligned columns) + row partials (2 strips)
    return 256 * 8 + sizeof(PilotOut) * (size_t)n + sizeof(ItemOut) * (size_t)n * ST_KMAX +
           2 * sizeof(uint32_t) * (size_t)n * ST_KMAX * 2048 + 2 * sizeof(uint32_t) * (size_t)n * 2 * H;
}

template <int VPL>
static int launch_stream(epid_ctx* ctx, cudaStream_t stream, int grid, size_t smem, const StreamGeom& sg, const FrameRef* refs, const PilotOut* pilot,
                         int nitems, ItemOut* items, uint32_t* col_raw, uint32_t* col_cl, uint32_t* row_raw, uint32_t* row_cl) {
    EPID_SMEM_OPT_IN(ctx, k_pf_stream<VPL>, smem);
    k_pf_stream<VPL><<<grid, ST_THREADS, smem, stream>>>(sg, refs, pilot, nitems, items, col_raw, col_cl, row_raw, row_cl);
    return EPID_OK;
}

int launch_pf_front(epid_ctx* ctx, cudaStream_t stream, const PfConst* d_cst, const StatsGeom& g, const FrameRef* refs, int n, PfFrame* fr,
                    FrameStats* stats, int* counters, void* scratch, PfTimers* tm) {
    const int H = g.H, W = g.W;
    StreamGeom sg;
    sg.H = H;
    sg.W = W;
    sg.nvec = (W + 7 + 7) / 8;          // worst-case misalignment of 7 pixels
    const int vpl = stream_vpl(sg.nvec, &sg.nstrips);
    sg.wa = sg.nstrips * vpl * 256;
    sg.row_bytes = sg.nvec * 16;
    sg.rps = ST_NCW / sg.nstrips;
    // items per frame: enough work items to balance the persistent grid (>= ~7 per CTA), rows per item <= ST_MAXROWS
    int K = (H + ST_MAXROWS - 1) / ST_MAXROWS;
    while (K < ST_KMAX && (long long)n * K < 7LL * ctx->sm_count) K *= 2;
    if (K > ST_KMAX) K = ST_KMAX;
    sg.K = K;
    sg.rows_per_item = (H + K - 1) / K;
    const int nitems = n * K;
    // carve the scratch area
    char* p = (char*)scratch;
    auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) / 256 * 256; return r; };
    PilotOut* pilot = (PilotOut*)take(sizeof(PilotOut) * (size_t)n);
    ItemOut* items = (ItemOut*)take(sizeof(ItemOut) * (size_t)nitems);
    uint32_t* col_raw = (uint32_t*)take(sizeof(uint32_t) * (size_t)nitems * sg.wa);
    uint32_t* col_cl = (uint32_t*)take(sizeof(uint32_t) * (size_t)nitems * sg.wa);
    uint32_t* row_raw = (uint32_t*)take(sizeof(uint32_t) * (size_t)n * 2 * H);
    uint32_t* row_cl = (uint32_t*)take(sizeof(uint32_t) * (size_t)n * 2 * H);

    k_pf_pilot<<<n, PILOT_THREADS, 0, stream>>>(g, refs, n, pilot);
    ctx->launches++;
    const size_t smem = 256 + (size_t)ST_NST * sg.rps * sg.row_bytes + sizeof(uint32_t) * (size_t)ST_NCW * vpl * 256;
    const int grid = nitems < ctx->sm_count ? nitems : ctx->sm_count;
    int rc = EPID_OK;
    if (tm) { rc = tm->mark(stream, PF_STAGE_INIT_PILOT); if (rc != EPID_OK) return rc; }
    if (tm && tm->on) { rc = tm->record(stream); if (rc != EPID_OK) return rc; }
    switch (vpl) {
        case 1: rc = launch_stream<1>(ctx, stream, grid, smem, sg, refs, pilot, nitems, items, col_raw, col_cl, row_raw, row_cl); break;
        case 2: rc = launch_stream<2>(ctx, stream, grid, smem, sg, refs, pilot, nitems, items, col_raw, col_cl, row_raw, row_cl); break;
        case 3: rc = launch_stream<3>(ctx, stream, grid, smem, sg, refs, pilot, nitems, items, col_raw, col_cl, row_raw, row_cl); break;
        default: rc = launch_stream<4>(ctx, stream, grid, smem, sg, refs, pilot, nitems, items, col_raw, col_cl, row_raw, row_cl); break;
    }
    if (rc != EPID_OK) return rc;
    ctx->launches++;
    if (tm && tm->on) { rc = tm->record(stream); if (rc != EPID_OK) return rc; }
    if (tm) { rc = tm->mark(stream, PF_STAGE_STREAM); if (rc != EPID_OK) return rc; }
    {
        const size_t tsm = pf_tail_smem_bytes(H, W);
        EPID_SMEM_OPT_IN(ctx, k_pf_tail, tsm);
        k_pf_tail<<<n, TAIL_THREADS, tsm, stream>>>(d_cst, g, sg, refs, pilot, items, col_raw, col_cl, row_raw, row_cl, fr, stats, counters);
        ctx->launches++;
        if (tm) { rc = tm->mark(stream, PF_STAGE_TAIL); if (rc != EPID_OK) return rc; }
    }
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace epid
