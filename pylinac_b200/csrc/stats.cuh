// Frame-statistics kernel interface (internal).
#pragma once
#include <cmath>

#include "common.cuh"

namespace epid {

constexpr int STATS_THREADS = 1024;
constexpr int STATS_MAX_RANKS = 16;
constexpr int STATS_MAX_DIM = 4096;  // rows / columns of the analysed view

// A frame view in HBM: `origin` points at pixel (0,0) of the analysed view (crop is a pointer offset,
// core/image.py:714-745), `pitch` = elements between rows.  If pitch % 8 == 0 the 8-pixel vectors of every row
// share one misalignment (origin address / 2) % 8 and 128-bit loads are legal on the aligned grid.
struct FrameRef {
    const uint16_t* origin;
    int pitch;
    int pad;
};

// refs[i] = view (r0, c0) of frame i of a contiguous batch of n frames of H0 x W0 pixels (pitch W0); one counted launch
void launch_refs_from_batch(epid_ctx* ctx, cudaStream_t stream, const uint16_t* base, int n, int H0, int W0, int r0, int c0, FrameRef* refs);

struct StatsGeom {   // identical for every frame of one launch
    int H, W;        // view size
    int vprp;        // (max) vectors per row, rounded up to a multiple of 32
    int groups;      // row groups handled concurrently = STATS_THREADS / vprp
    // corner boxes of BaseImage.check_inversion (core/image.py:881-894); box <= 0 disables
    int box, rp, cp;
    int nranks;
    uint32_t ranks[STATS_MAX_RANKS];  // 0-based order-statistic indices, ascending not required
};

struct FrameStats {  // per frame, device memory
    uint32_t mn, mx;
    uint32_t npix;
    uint32_t inv_certified;      // 0: ostat holds exact order statistics; 2 + inverted: inversion decision certified from counts
    unsigned long long sum;
    unsigned long long corner_sum;  // sum over the four corner boxes
    uint32_t ostat[STATS_MAX_RANKS];
};

// np.percentile(a, q_percent) with method="linear" over n values reads the sorted values at ranks prev and next and interpolates with
// gamma.  numpy's virtual index for "linear" is (n - 1) * q with q = q_percent / 100; written any other way it rounds differently for
// some (n, q) and the percentile moves by many ulps.  An index at or past n - 1 takes the last value, one below 0 the first.  F is the
// type numpy plans in: double, or float for a float32 array (q / float32(100), then (n - 1) * q, both in float32).
template <typename F> struct PctPlanOf { int prev, next; F gamma; };
using PctPlan = PctPlanOf<double>;

template <typename F>
__host__ __device__ inline PctPlanOf<F> pct_plan(int n, F q_percent) {
    const F vi = (F)(n - 1) * (q_percent / (F)100.0);
    PctPlanOf<F> p;
    if (vi >= (F)(n - 1)) {
        p.prev = p.next = n - 1;
        p.gamma = 0.0;
    } else if (vi < (F)0.0) {
        p.prev = p.next = 0;
        p.gamma = 0.0;
    } else {
        const F prev = floor(vi);
        p.prev = (int)prev;
        p.next = p.prev + 1;
        p.gamma = vi - prev;
    }
    return p;
}

// numpy _lerp (numpy/lib/_function_base_impl.py): a + (b-a)*t, and b - (b-a)*(1-t) where t >= 0.5; with pct_plan the two halves of
// np.percentile(method="linear").  np_lerp_d takes d = b - a as numpy formed it: an integer array subtracts in its own type.
template <typename F>
__host__ __device__ __forceinline__ F np_lerp_d(F a, F b, F d, F t) {
    F r = a + d * t;
    if (t >= (F)0.5) r = b - d * ((F)1.0 - t);
    return r;
}
__host__ __device__ __forceinline__ double np_lerp(double a, double b, double t) { return np_lerp_d(a, b, b - a, t); }

int make_stats_geom(StatsGeom* g, int H, int W);

// Exact statistics of frames d_frames[0..n): frame i writes d_stats[i]; rowsum: [i][H] u32, colsum: [i][W] u32 (may be null).
int launch_frame_stats(epid_ctx* ctx, cudaStream_t stream, const StatsGeom& g, const FrameRef* d_frames, int n, FrameStats* d_stats,
                       uint32_t* d_rowsum, uint32_t* d_colsum);
// Exact 65536-bin histogram of each frame's g.H x g.W view into d_hist[i][65536].  Only g.H and g.W are read: any view width.
int launch_frame_histogram(epid_ctx* ctx, cudaStream_t stream, const StatsGeom& g, const FrameRef* d_frames, int n, uint32_t* d_hist);
// check_inversion_by_histogram statistics (three percentile pairs in g.ranks): min / max / sum / row / column sums exactly; the decision
// certified from exact counts (FrameStats.inv_certified = 2 + inverted) or, where the bounds overlap, exact order statistics
// (inv_certified = 0)
int launch_frame_stats_inversion(epid_ctx* ctx, cudaStream_t stream, const StatsGeom& g, const FrameRef* d_frames, int n, FrameStats* d_stats,
                                 uint32_t* d_rowsum, uint32_t* d_colsum);
// the decision of check_inversion_by_histogram from a FrameStats record of either kind
__device__ __forceinline__ int stats_hist_inverted(const FrameStats& fs, double g_low, double g_mid, double g_high) {
    if (fs.inv_certified >= 2u) return (int)(fs.inv_certified - 2u);
    const double p_low = np_lerp((double)fs.ostat[0], (double)fs.ostat[1], g_low);
    const double p_mid = np_lerp((double)fs.ostat[2], (double)fs.ostat[3], g_mid);
    const double p_high = np_lerp((double)fs.ostat[4], (double)fs.ostat[5], g_high);
    return fabs(p_mid - p_low) > fabs(p_mid - p_high) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ exact 65536-bin histograms
// Shared-memory cache of histogram bins in front of a global histogram h.  Lanes of a warp that hold the same value are merged
// (__match_any_sync), and the merged count goes to slot value mod HIST_SLOTS, which the first value that claims it owns for the CTA's
// lifetime: EPID frames use a narrow band of values locally, so nearly every add stays in shared memory.  Values that lose a slot go
// straight to h.  The flush (after a __syncthreads) adds each occupied slot to h with one global atomic.
constexpr int HIST_SLOTS = 4096;
struct HistCache {
    uint32_t tag[HIST_SLOTS];    // value + 1, 0 = free
    uint32_t cnt[HIST_SLOTS];
};

__device__ __forceinline__ void hist_cache_init(HistCache& c) {
    for (int i = threadIdx.x; i < HIST_SLOTS; i += blockDim.x) { c.tag[i] = 0; c.cnt[i] = 0; }
}

// called by all 32 lanes of a warp; `in`: the lane holds a pixel v
__device__ __forceinline__ void hist_cache_add(HistCache& c, uint32_t* h, uint32_t v, bool in) {
    const unsigned m = __match_any_sync(0xffffffffu, in ? v : 0x10000u);
    if (in && (int)(threadIdx.x & 31) == __ffs(m) - 1) {
        const uint32_t cn = (uint32_t)__popc(m), slot = v & (HIST_SLOTS - 1);
        const uint32_t old = atomicCAS(&c.tag[slot], 0u, v + 1u);
        if (old == 0u || old == v + 1u) atomicAdd(&c.cnt[slot], cn);
        else atomicAdd(&h[v], cn);
    }
}

__device__ __forceinline__ void hist_cache_flush(const HistCache& c, uint32_t* h) {
    for (int i = threadIdx.x; i < HIST_SLOTS; i += blockDim.x) {
        const uint32_t tg = c.tag[i];
        if (tg) atomicAdd(&h[tg - 1u], c.cnt[i]);
    }
}

// Order statistics of a 65536-bin histogram, by a CTA of HIST_RANK_THREADS threads that each own 256 consecutive bins: the bin count of
// each thread, a serial exclusive prefix over the 256 partials, then the owner of each rank walks its bins.  ranks[0..nr) (0-based,
// any order) -> s.values; s.first / s.last = first / last non-empty bin; wsum (optional, HIST_RANK_THREADS entries): sum of bin * count
// per thread.  HistPtr is `const volatile uint32_t*` where threads of the CTA update the histogram between searches.  Every thread of
// the CTA calls it; the results are read after its closing barrier.
constexpr int HIST_RANK_THREADS = 256;
struct HistRanks {
    uint32_t part[HIST_RANK_THREADS];
    uint32_t values[STATS_MAX_RANKS];
    uint32_t first, last;
};

template <typename HistPtr>
__device__ __forceinline__ void hist_rank_search(HistPtr hist, const uint32_t* ranks, int nr, HistRanks& s, unsigned long long* wsum = nullptr) {
    const int tid = threadIdx.x;
    const int b0 = tid * (65536 / HIST_RANK_THREADS), b1 = b0 + 65536 / HIST_RANK_THREADS;
    uint32_t c = 0, lo_bin = 0xffffffffu, hi_bin = 0;
    unsigned long long ws = 0;
    for (int b = b0; b < b1; b++) {
        const uint32_t hb = hist[b];
        c += hb;
        if (wsum) ws += (unsigned long long)hb * (unsigned)b;
        if (hb) { if (lo_bin == 0xffffffffu) lo_bin = b; hi_bin = b; }
    }
    s.part[tid] = c;
    if (wsum) wsum[tid] = ws;
    if (tid == 0) { s.first = 0xffffffffu; s.last = 0; }
    __syncthreads();
    if (lo_bin != 0xffffffffu) { atomicMin(&s.first, lo_bin); atomicMax(&s.last, hi_bin); }
    uint32_t excl = 0;
    for (int k = 0; k < tid; k++) excl += s.part[k];
    for (int r = 0; r < nr; r++) {
        const uint32_t rk = ranks[r];
        if (rk >= excl && rk < excl + c) {
            uint32_t acc = excl;
            for (int b = b0; b < b1; b++) {
                const uint32_t hb = hist[b];
                if (rk < acc + hb) { s.values[r] = (uint32_t)b; break; }
                acc += hb;
            }
        }
    }
    __syncthreads();
}

}  // namespace epid
