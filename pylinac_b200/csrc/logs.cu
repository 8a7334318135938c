// Machine-log fluence maps and the per-frame pieces of the fluence gamma (log_analyzer.py:478-612, 690-758).
//
// FluenceBase.calc_map builds one float32 "line" per leaf pair: for every beam-on snapshot s (in order) the columns between the
// pair's leaf / jaw edges get `line[a:b] += MU_differential[s]` (numpy: (float)((double)line + mu_diff), a double rounding), a
// pair that did not move gets `line[a:b] = float32(MU_total)` once.  The line is written to row pair - 1 (or, with equal_aspect,
// to the pair's row range) of a float64 map; a Dynalog map (MU_total == 25000) is divided by MU_total.
//
// Device input (one layout for both log formats): every log is a column table inside one host arena, copied to the device once.
// Value (snapshot s, column c) sits at  data_off + (s * snap_stride + c * col_stride) * elem  with elem 4 (a trajectory log's raw
// float32 body, widened to fp64 on load: snap_stride = 2 * sum(samples_per_axis), col_stride = 1) or 8 (a Dynalog's fp64 columns,
// built on the host from the text: snap_stride = 1, col_stride = num_snapshots).  The host passes the beam-on snapshot list and the
// per-pair decisions the reference makes with numpy (moving_leaves, leaf_under_y_jaw) and the row bounds of every pair.
//
//   k_log_fluence   CTA per (pair, log, kind): the integer edges of a chunk of beam-on snapshots are computed once into shared
//                   memory; each thread owns columns (float32 accumulators in registers) and walks the chunk in snapshot order, so
//                   every pixel sees the reference's summation order.  Work per pixel and snapshot: one compare, one add if covered.
//
// Fluence gamma (BaseImage.gamma on the two fluence maps, core/image.py:928-1017): check_inversion_by_histogram of a float64 frame
// needs np.percentile(a, 5 / 50 / 95) exactly, so
//   k_sel_hist / k_sel_pick   8 passes of an 8-bit radix select of the order statistics 0, n-1 and the (prev, next) ranks of the
//                             three percentiles, on the order-preserving uint64 image of each double
//   k_inv_apply               the decision and, where it holds, the reference's invert (-a + max + min)
// then the existing epid_ground / epid_normalize / epid_gamma, and
//   k_gstat_partial / _final  per frame: sum and count of the non-nan gamma values, count below 1 (nanmean, pass percent)
#include <cmath>

#include "stats.cuh"

namespace epid {
namespace {

constexpr int LF_THREADS = 256;
constexpr int LF_COLS = 16;                  // columns per thread and column group: LF_THREADS * LF_COLS = 4096 (res >= 0.1 mm: one group)
constexpr int LF_CHUNK = 1024;               // beam-on snapshots staged in shared memory at a time

struct LogDesc {
    int64_t data_off;                        // byte offset of the log's column table in the arena
    int64_t snap_stride, col_stride;         // in elements
    int32_t f64;                             // 1: float64 values, 0: float32
    int32_t nsnap;
    int32_t col_mu[2];                       // [actual, expected] MU column
    int32_t col_x1, col_x2;                  // jaw X1 / X2, actual
    int32_t col_leaf[2];                     // [actual, expected] column of leaf 1; leaf l at col_leaf + 2 (l - 1)
    int32_t num_pairs;
    int32_t snap_off, nbeam;                 // beam-on snapshot indices snaps[snap_off .. snap_off + nbeam)
    int32_t pair_off;                        // PF_* flags of pair p at pflags[pair_off + p - 1]
    int32_t row_off;                         // output rows [rows[row_off + 2 (p - 1)], rows[row_off + 2 (p - 1) + 1]) of pair p
    int32_t flags[2];                        // per kind: LF_ZERO (whole map stays 0), LF_DIV25000 (map / MU_total)
    int32_t pad;
};
static_assert(sizeof(LogDesc) == 88, "LogDesc layout is shared with the host (log_analyzer.py LOG_DESC_DTYPE)");

enum { LF_ZERO = 1, LF_DIV25000 = 2 };
enum { PF_UNDER_JAW = 1, PF_MOVED = 2 };

__device__ __forceinline__ double ld(const uint8_t* arena, const LogDesc& d, int64_t s, int64_t c) {
    const int64_t i = s * d.snap_stride + c * d.col_stride;
    return d.f64 ? reinterpret_cast<const double*>(arena + d.data_off)[i] : (double)reinterpret_cast<const float*>(arena + d.data_off)[i];
}

// numpy's min / max reductions: nan propagates
__device__ __forceinline__ double nan_min(double a, double b) { return (isnan(a) || isnan(b)) ? NAN : (b < a ? b : a); }
__device__ __forceinline__ double nan_max(double a, double b) { return (isnan(a) || isnan(b)) ? NAN : (b > a ? b : a); }

// Python slice bound of a sequence of length W: negative wraps by +W, then clipped to [0, W] (v is integer-valued)
__device__ __forceinline__ int slice_bound(double v, int W) {
    if (v < 0.0) v += (double)W;
    if (v < 0.0) v = 0.0;
    if (v > (double)W) v = (double)W;
    return (int)v;
}

// int(max(lt_mlc, lt_jaw)) / int(min(rt_mlc, rt_jaw)) with Python's max / min (the first argument unless the second is strictly
// beyond it); the operands are np.round results, so int() is exact
__device__ __forceinline__ void pair_edges(double xr, double xl, double x1, double x2, double res, double pos_off, double h200, int W, int& a,
                                           int& b) {
    const double rt_mlc = rint((xr * 10.0) / res) + pos_off;
    const double lt_mlc = -rint((xl * 10.0) / res) + pos_off;
    const double lt_jaw = rint(h200 - (x1 * 10.0) / res);
    const double rt_jaw = rint((x2 * 10.0) / res + h200);
    const double l = lt_jaw > lt_mlc ? lt_jaw : lt_mlc;
    const double r = rt_jaw < rt_mlc ? rt_jaw : rt_mlc;
    a = slice_bound(trunc(l), W);
    b = slice_bound(trunc(r), W);
}

__global__ void __launch_bounds__(LF_THREADS) k_log_fluence(const uint8_t* __restrict__ arena, const LogDesc* __restrict__ logs,
                                                            const int32_t* __restrict__ snaps, const uint8_t* __restrict__ pflags,
                                                            const int32_t* __restrict__ rows, double res, int W, int R, int kinds,
                                                            double* __restrict__ out_actual, double* __restrict__ out_expected) {
    __shared__ int s_a[LF_CHUNK], s_b[LF_CHUNK];
    __shared__ double s_mu[LF_CHUNK];
    __shared__ double s_red[2][LF_THREADS / 32];
    const int pair = blockIdx.x + 1, li = blockIdx.y, kind = blockIdx.z;   // kind 0: actual, 1: expected
    if (!((kinds >> kind) & 1)) return;
    const LogDesc d = logs[li];
    const int kflags = kind ? d.flags[1] : d.flags[0];
    if (pair > d.num_pairs || (kflags & LF_ZERO)) return;
    const uint8_t pf = pflags[d.pair_off + pair - 1];
    if (pf & PF_UNDER_JAW) return;
    double* out = (kind == 0 ? out_actual : out_expected) + (size_t)li * R * W;
    const int r0 = rows[d.row_off + 2 * (pair - 1)], r1 = rows[d.row_off + 2 * (pair - 1) + 1];
    const double pos_off = rint(200.0 / res), h200 = 200.0 / res;
    const int64_t c_leaf = kind ? d.col_leaf[1] : d.col_leaf[0];
    const int64_t c_right = c_leaf + 2 * (pair - 1), c_left = c_leaf + 2 * (pair - 1 + d.num_pairs);
    const int64_t c_mu = kind ? d.col_mu[1] : d.col_mu[0];
    const double mu_total = ld(arena, d, d.nsnap - 1, c_mu);
    const double scale = (kflags & LF_DIV25000) ? mu_total : 1.0;
    const int tid = threadIdx.x;

    if (!(pf & PF_MOVED)) {
        // static pair: the first beam-on snapshot's leaves against the extreme jaw edges over ALL snapshots (ndarray.min / max:
        // a nan sample makes the extreme nan, and Python's max / min below then keep the leaf edge)
        double mn = INFINITY, mx = -INFINITY;
        for (int s = tid; s < d.nsnap; s += LF_THREADS) {
            mn = nan_min(mn, rint(h200 - (ld(arena, d, s, d.col_x1) * 10.0) / res));
            mx = nan_max(mx, rint((ld(arena, d, s, d.col_x2) * 10.0) / res + h200));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = nan_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if ((tid & 31) == 0) { s_red[0][tid >> 5] = mn; s_red[1][tid >> 5] = mx; }
        __syncthreads();
        mn = s_red[0][0];
        mx = s_red[1][0];
        for (int k = 1; k < LF_THREADS / 32; k++) { mn = nan_min(mn, s_red[0][k]); mx = nan_max(mx, s_red[1][k]); }
        const int s0 = snaps[d.snap_off];
        const double rt_mlc = rint((ld(arena, d, s0, c_right) * 10.0) / res) + pos_off;
        const double lt_mlc = -rint((ld(arena, d, s0, c_left) * 10.0) / res) + pos_off;
        const double l = mn > lt_mlc ? mn : lt_mlc, r = mx < rt_mlc ? mx : rt_mlc;
        const int a = slice_bound(trunc(l), W), b = slice_bound(trunc(r), W);
        const double v = (double)(float)mu_total / scale;
        for (int row = r0; row < r1; row++)
            for (int c = tid; c < W; c += LF_THREADS) out[(size_t)row * W + c] = (c >= a && c < b) ? v : 0.0;
        return;
    }

    for (int cg = 0; cg < W; cg += LF_THREADS * LF_COLS) {
        const int nk = min(LF_COLS, (W - cg + LF_THREADS - 1) / LF_THREADS);     // column slots of this group inside the map
        float acc[LF_COLS];
#pragma unroll
        for (int k = 0; k < LF_COLS; k++) acc[k] = 0.0f;
        for (int j0 = 0; j0 < d.nbeam; j0 += LF_CHUNK) {
            const int m = min(LF_CHUNK, d.nbeam - j0);
            __syncthreads();
            for (int j = tid; j < m; j += LF_THREADS) {
                const int s = snaps[d.snap_off + j0 + j];
                int a, b;
                pair_edges(ld(arena, d, s, c_right), ld(arena, d, s, c_left), ld(arena, d, s, d.col_x1), ld(arena, d, s, d.col_x2), res,
                           pos_off, h200, W, a, b);
                s_a[j] = a;
                s_b[j] = b;
                const double mu = ld(arena, d, s, c_mu);
                s_mu[j] = s == 0 ? mu : mu - ld(arena, d, s - 1, c_mu);     // [mu[0]] + np.diff(mu)
            }
            __syncthreads();
            for (int j = 0; j < m; j++) {
                const int a = s_a[j], b = s_b[j];
                const double dm = s_mu[j];
#pragma unroll
                for (int k = 0; k < LF_COLS; k++) {
                    if (k >= nk) break;
                    const int c = cg + k * LF_THREADS + tid;
                    if (c >= a && c < b) acc[k] = (float)((double)acc[k] + dm);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < LF_COLS; k++) {
            const int c = cg + k * LF_THREADS + tid;
            if (c < W) {
                const double v = (double)acc[k] / scale;
                for (int row = r0; row < r1; row++) out[(size_t)row * W + c] = v;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ exact order statistics
constexpr int SEL_RANKS = 8;                 // 0, n - 1, (prev, next) of the 5th, 50th and 95th percentile
constexpr int SEL_THREADS = 256;
constexpr int SEL_BLOCKS = 32;               // CTAs per frame and pass

__device__ __forceinline__ uint64_t okey(double v) {      // order-preserving image of a double (nan-free input)
    const uint64_t u = (uint64_t)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double okey_value(uint64_t k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

struct SelState {
    uint64_t prefix[SEL_RANKS];              // the key bits decided so far
    uint32_t rank[SEL_RANKS];                // remaining rank inside the prefix's bucket
};

__global__ void __launch_bounds__(SEL_THREADS) k_sel_hist(const double* __restrict__ data, size_t per_frame, const SelState* __restrict__ st,
                                                          int shift, uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[SEL_RANKS][256];
    __shared__ uint64_t pre[SEL_RANKS];
    const int f = blockIdx.y;
    for (int i = threadIdx.x; i < SEL_RANKS * 256; i += SEL_THREADS) (&h[0][0])[i] = 0;
    if (threadIdx.x < SEL_RANKS) pre[threadIdx.x] = st[f].prefix[threadIdx.x];
    __syncthreads();
    const double* a = data + (size_t)f * per_frame;
    const int hs = shift + 8;
    for (size_t i = (size_t)blockIdx.x * SEL_THREADS + threadIdx.x; i < per_frame; i += (size_t)SEL_BLOCKS * SEL_THREADS) {
        const uint64_t k = okey(a[i]);
        const uint32_t dig = (uint32_t)(k >> shift) & 255u;
#pragma unroll
        for (int r = 0; r < SEL_RANKS; r++)
            if (hs >= 64 || (k >> hs) == (pre[r] >> hs)) atomicAdd(&h[r][dig], 1u);
    }
    __syncthreads();
    uint32_t* g = hist + (size_t)f * SEL_RANKS * 256;
    for (int i = threadIdx.x; i < SEL_RANKS * 256; i += SEL_THREADS)
        if ((&h[0][0])[i]) atomicAdd(g + i, (&h[0][0])[i]);
}

// one warp per rank: the digit whose bucket holds the remaining rank; clears the histogram for the next pass
__global__ void k_sel_pick(SelState* __restrict__ st, int shift, uint32_t* __restrict__ hist) {
    const int f = blockIdx.x, r = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* g = hist + ((size_t)f * SEL_RANKS + r) * 256;
    uint32_t c[8], tot = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { c[k] = g[lane * 8 + k]; tot += c[k]; g[lane * 8 + k] = 0; }
    uint32_t incl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    const uint32_t want = st[f].rank[r];
    uint32_t base = incl - tot;
    if (want >= base && want < incl) {
        for (int k = 0; k < 8; k++) {
            if (want < base + c[k]) {
                st[f].prefix[r] |= (uint64_t)(lane * 8 + k) << shift;
                st[f].rank[r] = want - base;
                break;
            }
            base += c[k];
        }
    }
}

__global__ void k_sel_init(SelState* st, int n, uint32_t npix, const uint32_t* __restrict__ ranks) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    for (int r = 0; r < SEL_RANKS; r++) { st[f].prefix[r] = 0; st[f].rank[r] = ranks[r]; }
}

struct InvPlan { double g_low, g_mid, g_high; };

// check_inversion_by_histogram (core/image.py:899-926) and invert (core/array_utils.py:75-77): -a + max + min
__global__ void k_inv_apply(const double* __restrict__ in, double* __restrict__ out, size_t per_frame, const SelState* __restrict__ st, InvPlan p,
                            int32_t* __restrict__ inverted) {
    const int f = blockIdx.y;
    double v[SEL_RANKS];
#pragma unroll
    for (int r = 0; r < SEL_RANKS; r++) v[r] = okey_value(st[f].prefix[r]);
    const double p_low = np_lerp(v[2], v[3], p.g_low), p_mid = np_lerp(v[4], v[5], p.g_mid), p_high = np_lerp(v[6], v[7], p.g_high);
    const bool inv = fabs(p_mid - p_low) > fabs(p_mid - p_high);
    if (blockIdx.x == 0 && threadIdx.x == 0 && inverted) inverted[f] = inv ? 1 : 0;
    const double mn = v[0], mx = v[1];
    const double* a = in + (size_t)f * per_frame;
    double* o = out + (size_t)f * per_frame;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_frame; i += (size_t)gridDim.x * blockDim.x)
        o[i] = inv ? (-a[i] + mx) + mn : a[i];
}

// ------------------------------------------------------------------------------------------------ gamma statistics
constexpr int GS_THREADS = 256, GS_BLOCKS = 64;

__global__ void __launch_bounds__(GS_THREADS) k_gstat_partial(const double* __restrict__ g, size_t per_frame, double* __restrict__ psum,
                                                              unsigned long long* __restrict__ pcnt, unsigned long long* __restrict__ ppass) {
    __shared__ double ss[GS_THREADS / 32];
    __shared__ unsigned long long sc[GS_THREADS / 32], sp[GS_THREADS / 32];
    const int f = blockIdx.y;
    const double* a = g + (size_t)f * per_frame;
    double s = 0.0;
    unsigned long long cnt = 0, pass = 0;
    for (size_t i = (size_t)blockIdx.x * GS_THREADS + threadIdx.x; i < per_frame; i += (size_t)GS_BLOCKS * GS_THREADS) {
        const double v = a[i];
        if (!isnan(v)) { s += v; cnt++; if (v < 1.0) pass++; }
    }
    s = warp_sum(s);
    cnt = warp_sum(cnt);
    pass = warp_sum(pass);
    if ((threadIdx.x & 31) == 0) { ss[threadIdx.x >> 5] = s; sc[threadIdx.x >> 5] = cnt; sp[threadIdx.x >> 5] = pass; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        unsigned long long c = 0, q = 0;
        for (int k = 0; k < GS_THREADS / 32; k++) { t += ss[k]; c += sc[k]; q += sp[k]; }
        psum[f * GS_BLOCKS + blockIdx.x] = t;
        pcnt[f * GS_BLOCKS + blockIdx.x] = c;
        ppass[f * GS_BLOCKS + blockIdx.x] = q;
    }
}

__global__ void k_gstat_final(const double* __restrict__ psum, const unsigned long long* __restrict__ pcnt, const unsigned long long* __restrict__ ppass,
                              int n, double* __restrict__ sum, int64_t* __restrict__ cnt, int64_t* __restrict__ pass) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    double t = 0.0;
    unsigned long long c = 0, q = 0;
    for (int k = 0; k < GS_BLOCKS; k++) { t += psum[f * GS_BLOCKS + k]; c += pcnt[f * GS_BLOCKS + k]; q += ppass[f * GS_BLOCKS + k]; }
    sum[f] = t;
    cnt[f] = (int64_t)c;
    pass[f] = (int64_t)q;
}

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

int sync_or_fail(epid_ctx* ctx, const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { set_error("%s: %s", what, cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_log_fluence(epid_ctx* ctx, const void* arena, size_t arena_bytes, const void* logs, int32_t n, const int32_t* snaps,
                                    int32_t n_snaps, const uint8_t* pair_flags, int32_t n_pair_flags, const int32_t* rows, int32_t n_rows,
                                    double resolution, int32_t w, int32_t h, int32_t kinds, epid_batch** out_actual, epid_batch** out_expected) {
    EPID_REQUIRE(ctx && arena && logs && pair_flags && rows && out_actual && out_expected, EPID_ERR_INVALID, "NULL argument");
    *out_actual = *out_expected = nullptr;
    EPID_REQUIRE(n > 0 && n <= 65535, EPID_ERR_INVALID, "n = %d logs (1 .. 65535 per call)", n);
    EPID_REQUIRE(w > 0 && h > 0 && resolution > 0.0, EPID_ERR_INVALID, "fluence map %d x %d at resolution %g", h, w, resolution);
    EPID_REQUIRE(kinds >= 1 && kinds <= 3, EPID_ERR_INVALID, "kinds must be 1 (actual), 2 (expected) or 3 (both)");
    EPID_REQUIRE(n_snaps >= 0 && (n_snaps == 0 || snaps), EPID_ERR_INVALID, "NULL beam-on snapshot list");
    const LogDesc* ld_ = (const LogDesc*)logs;
    int max_pairs = 0;
    for (int i = 0; i < n; i++) {
        const LogDesc& d = ld_[i];
        const int64_t esz = d.f64 ? 8 : 4;
        const int64_t last = (int64_t)(d.nsnap - 1) * d.snap_stride;
        const int maxc = max(max(max(d.col_mu[0], d.col_mu[1]), max(d.col_x1, d.col_x2)),
                             max(d.col_leaf[0], d.col_leaf[1]) + 2 * (2 * d.num_pairs - 1));
        EPID_REQUIRE(d.nsnap > 0 && d.num_pairs >= 0 && d.nbeam >= 0 && d.snap_off >= 0 && d.snap_off + d.nbeam <= n_snaps &&
                         d.pair_off >= 0 && d.pair_off + d.num_pairs <= n_pair_flags && d.row_off >= 0 && d.row_off + 2 * d.num_pairs <= n_rows &&
                         d.data_off >= 0 && (d.data_off % esz) == 0 && d.data_off + (last + (int64_t)maxc * d.col_stride + 1) * esz <= (int64_t)arena_bytes,
                     EPID_ERR_INVALID, "log %d: descriptor outside the arena / lists", i);
        bool live = false;                     // a requested kind whose map is computed needs beam-on snapshots
        for (int k = 0; k < 2; k++) live = live || (((kinds >> k) & 1) && !(d.flags[k] & LF_ZERO));
        EPID_REQUIRE(d.nbeam > 0 || !live, EPID_ERR_INVALID, "log %d: no beam-on snapshots", i);
        for (int j = 0; j < d.nbeam; j++)
            EPID_REQUIRE(snaps[d.snap_off + j] >= 0 && snaps[d.snap_off + j] < d.nsnap, EPID_ERR_INVALID, "log %d: snapshot index out of range", i);
        for (int p = 0; p < 2 * d.num_pairs; p++)
            EPID_REQUIRE(rows[d.row_off + p] >= 0 && rows[d.row_off + p] <= h, EPID_ERR_INVALID, "log %d: row bound outside [0, %d]", i, h);
        max_pairs = max(max_pairs, d.num_pairs);
    }
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t sz_arena = al256(arena_bytes), sz_logs = al256(sizeof(LogDesc) * n), sz_snaps = al256(4 * (size_t)max(n_snaps, 1));
    const size_t sz_pf = al256((size_t)max(n_pair_flags, 1)), sz_rows = al256(4 * (size_t)max(n_rows, 1));
    int rc = ensure_scratch(ctx, sz_arena + sz_logs + sz_snaps + sz_pf + sz_rows);
    if (rc != EPID_OK) return rc;
    char* p = (char*)ctx->scratch;
    uint8_t* d_arena = (uint8_t*)p; p += sz_arena;
    LogDesc* d_logs = (LogDesc*)p; p += sz_logs;
    int32_t* d_snaps = (int32_t*)p; p += sz_snaps;
    uint8_t* d_pf = (uint8_t*)p; p += sz_pf;
    int32_t* d_rows = (int32_t*)p;
    epid_batch* outs[2] = {nullptr, nullptr};
    for (int k = 0; k < 2; k++) {
        if (!((kinds >> k) & 1)) continue;
        rc = epid_batch_alloc(ctx, EPID_F64, n, h, w, &outs[k]);
        if (rc != EPID_OK) { epid_batch_free(outs[0]); return rc; }
    }
    cudaStream_t s = ctx->stream;
    cudaError_t e = cudaMemcpyAsync(d_arena, arena, arena_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_logs, logs, sizeof(LogDesc) * n, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && n_snaps) e = cudaMemcpyAsync(d_snaps, snaps, 4 * (size_t)n_snaps, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && n_pair_flags) e = cudaMemcpyAsync(d_pf, pair_flags, (size_t)n_pair_flags, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && n_rows) e = cudaMemcpyAsync(d_rows, rows, 4 * (size_t)n_rows, cudaMemcpyHostToDevice, s);
    for (int k = 0; k < 2 && e == cudaSuccess; k++)
        if (outs[k]) e = cudaMemsetAsync(outs[k]->dptr, 0, outs[k]->bytes(), s);
    if (e == cudaSuccess && max_pairs > 0) {
        k_log_fluence<<<dim3(max_pairs, n, 2), LF_THREADS, 0, s>>>(d_arena, d_logs, d_snaps, d_pf, d_rows, resolution, w, h, kinds,
                                                                    outs[0] ? (double*)outs[0]->dptr : nullptr,
                                                                    outs[1] ? (double*)outs[1]->dptr : nullptr);
        ctx->launches++;
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        set_error("log fluence: %s", cudaGetErrorString(e));
        epid_batch_free(outs[0]);
        epid_batch_free(outs[1]);
        return EPID_ERR_CUDA;
    }
    *out_actual = outs[0];
    *out_expected = outs[1];
    return EPID_OK;
}

extern "C" int32_t epid_hist_invert(epid_ctx* ctx, const epid_batch* in, epid_batch** out, int32_t* inverted) {
    EPID_REQUIRE(ctx && in && out, EPID_ERR_INVALID, "NULL argument");
    *out = nullptr;
    EPID_REQUIRE(in->dtype == EPID_F64, EPID_ERR_UNSUPPORTED, "the float64 inversion check takes float64 frames");
    const size_t per = (size_t)in->h * in->w;
    EPID_REQUIRE(per <= 0xffffffffull, EPID_ERR_UNSUPPORTED, "frames of more than 2^32 pixels");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = in->n;
    const int npix = (int)per;
    const PctPlan lo = pct_plan(npix, 5.0), mid = pct_plan(npix, 50.0), hi = pct_plan(npix, 95.0);
    const uint32_t ranks[SEL_RANKS] = {0u, (uint32_t)(npix - 1), (uint32_t)lo.prev, (uint32_t)lo.next, (uint32_t)mid.prev, (uint32_t)mid.next,
                                       (uint32_t)hi.prev, (uint32_t)hi.next};
    const size_t sz_st = al256(sizeof(SelState) * n), sz_h = al256(4 * (size_t)n * SEL_RANKS * 256), sz_r = al256(sizeof(ranks));
    int rc = ensure_scratch(ctx, sz_st + sz_h + sz_r + al256(4 * (size_t)n));
    if (rc != EPID_OK) return rc;
    char* p = (char*)ctx->scratch;
    SelState* d_st = (SelState*)p; p += sz_st;
    uint32_t* d_hist = (uint32_t*)p; p += sz_h;
    uint32_t* d_ranks = (uint32_t*)p; p += sz_r;
    int32_t* d_inv = (int32_t*)p;
    rc = epid_batch_alloc(ctx, EPID_F64, n, in->h, in->w, out);
    if (rc != EPID_OK) return rc;
    cudaStream_t s = ctx->stream;
    cudaError_t e = cudaMemcpyAsync(d_ranks, ranks, sizeof(ranks), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_hist, 0, 4 * (size_t)n * SEL_RANKS * 256, s);
    if (e == cudaSuccess) {
        k_sel_init<<<(n + 127) / 128, 128, 0, s>>>(d_st, n, (uint32_t)npix, d_ranks);
        for (int shift = 56; shift >= 0; shift -= 8) {
            k_sel_hist<<<dim3(SEL_BLOCKS, n), SEL_THREADS, 0, s>>>((const double*)in->dptr, per, d_st, shift, d_hist);
            k_sel_pick<<<n, SEL_RANKS * 32, 0, s>>>(d_st, shift, d_hist);
        }
        int bx = (int)((per + 256 * 8 - 1) / (256 * 8));
        bx = max(1, min(bx, 1024));
        k_inv_apply<<<dim3(bx, n), 256, 0, s>>>((const double*)in->dptr, (double*)(*out)->dptr, per, d_st, InvPlan{lo.gamma, mid.gamma, hi.gamma}, d_inv);
        ctx->launches += 2 + 2 * 8;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && inverted) e = cudaMemcpyAsync(inverted, d_inv, 4 * (size_t)n, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        set_error("inversion check: %s", cudaGetErrorString(e));
        epid_batch_free(*out);
        *out = nullptr;
        return EPID_ERR_CUDA;
    }
    return EPID_OK;
}

extern "C" int32_t epid_gamma_stats(epid_ctx* ctx, const epid_batch* gamma, double* sum, int64_t* count, int64_t* passing) {
    EPID_REQUIRE(ctx && gamma && sum && count && passing, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(gamma->dtype == EPID_F64, EPID_ERR_UNSUPPORTED, "gamma statistics take a float64 gamma batch");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = gamma->n;
    const size_t per = (size_t)gamma->h * gamma->w;
    const size_t sz_p = al256(8 * (size_t)n * GS_BLOCKS), sz_o = al256(8 * (size_t)n);
    int rc = ensure_scratch(ctx, 3 * sz_p + 3 * sz_o);
    if (rc != EPID_OK) return rc;
    char* p = (char*)ctx->scratch;
    double* d_psum = (double*)p; p += sz_p;
    unsigned long long* d_pcnt = (unsigned long long*)p; p += sz_p;
    unsigned long long* d_ppass = (unsigned long long*)p; p += sz_p;
    double* d_sum = (double*)p; p += sz_o;
    int64_t* d_cnt = (int64_t*)p; p += sz_o;
    int64_t* d_pass = (int64_t*)p;
    cudaStream_t s = ctx->stream;
    k_gstat_partial<<<dim3(GS_BLOCKS, n), GS_THREADS, 0, s>>>((const double*)gamma->dptr, per, d_psum, d_pcnt, d_ppass);
    k_gstat_final<<<(n + 127) / 128, 128, 0, s>>>(d_psum, d_pcnt, d_ppass, n, d_sum, d_cnt, d_pass);
    ctx->launches += 2;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(sum, d_sum, 8 * (size_t)n, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(count, d_cnt, 8 * (size_t)n, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(passing, d_pass, 8 * (size_t)n, cudaMemcpyDeviceToHost, s);
    if (e != cudaSuccess) { set_error("gamma statistics: %s", cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    return sync_or_fail(ctx, "gamma statistics");
}
