// Batched FieldAnalysis.analyze() on the GPU.  One result per frame; frames never leave HBM between stages.
//
// Reference path reproduced (pylinac v3.46.0):
//   FieldAnalysis.__init__ / _determine_center / _extract_profiles / _analyze            field_analysis.py:445-864
//   _get_vert_values / _get_horiz_values                                                  field_analysis.py:1069-1117
//   protocol functions: flatness_dose_difference / flatness_dose_ratio / symmetry_*       field_analysis.py:37-231
//   SingleProfile: _interpolate, _normalize, beam_center, geometric_center, fwxm_data, field_data, inflection_data,
//                  penumbra, field_calculation                                            core/profile.py:1125-1937
//   MultiProfile.find_peaks / find_valleys, find_peaks                                    core/profile.py:2050-2110, 2545-2649
//   BaseImage.check_inversion_by_histogram, invert                                        core/image.py:899-926
// Third-party arithmetic restated (scipy 1.18.1 / numpy 2.3.5): interpolate.interp1d(kind='linear', 'extrapolate') =
// searchsorted + slope * (x - x_lo) + y_lo; np.interp; np.linspace; ndimage.gaussian_filter1d = symmetric correlate1d,
// mode='reflect', weights supplied by the binding; np.gradient; signal.find_peaks (peaks.cuh); stats.linregress;
// np.polyfit(deg=2) as least squares on centred / scaled abscissae.
// Scope: interpolation NONE / LINEAR, edge detection FWHM / INFLECTION_DERIVATIVE, every normalisation, protocols NONE /
// VARIAN / SIEMENS / ELEKTA.  SPLINE interpolation and INFLECTION_HILL are refused by the binding (NotImplementedError).
// Documented deviation: the "top" of the field is the exact vertex of the fitted parabola clipped to its window; the
// reference runs L-BFGS-B with a finite-difference gradient on the same parabola and stops wherever its rounding noise
// lets it (tests/test_oracle_field.py), so the top_* fields are outside the parity bar.
//
// Stages:
//   k_inv_* / k_hist_view  min / max + exact row and column sums of every frame; the p5 / p50 / p95 inversion decision,
//                    certified from exact counts or read from the exact histogram                                  (stats.cu)
//   k_field_center   CTA per (frame, axis): inversion decision, SingleProfile(sum profile).beam_center() -> strip position
//   k_field_strips   CTA per (frame, axis): mean over the strip of rows / columns -> raw profile
//   k_field_profile  CTA per (frame, axis): SingleProfile(profile, dpmm, ...) -> penumbra, centres, field sizes, slopes,
//                    top, protocol flatness / symmetry
#include <cmath>

#include "peaks.cuh"
#include "pf_common.cuh"

namespace epid {

constexpr int FA_THREADS = 256;
constexpr int FA_WARPS = FA_THREADS / 32;

struct FieldConst {
    epid_field_params p;
    int H, W;
    PctPlan p5, p50, p95;
    int nmax;                 // capacity of the per-(frame, axis) profile arrays
    int pcap;                 // capacity (power of two) of the per-(frame, axis) peak arrays
    size_t stride;            // doubles per (frame, axis) work area: 4 * nmax + 8 * pcap
    int lw[2];                // gaussian radius for the horizontal / vertical profile
    int n_expect[2];          // profile length the weights were made for
};

struct FieldFrame {
    uint32_t mn, mx;
    int flip;                 // pixels are read as flip ? mx + mn - v : v
    int hist_inverted;
    double pos[2];            // [0] horiz_position (ratio of H: where the horizontal profile is taken), [1] vert_position
    int lo[2], hi[2];         // strips: [0] rows [bottom, top), [1] columns [left, right)
};

// ------------------------------------------------------------------------------------------------ block helpers
struct BlockRed {
    double d[FA_WARPS + 1];
    int i[FA_WARPS + 1];
};

__device__ __forceinline__ double block_sum(double v, BlockRed* r) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) r->d[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
        for (int k = 0; k < FA_WARPS; k++) s += r->d[k];
        r->d[FA_WARPS] = s;
    }
    __syncthreads();
    return r->d[FA_WARPS];
}

__device__ __forceinline__ double block_min(double v, BlockRed* r) {
    v = warp_min(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) r->d[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = r->d[0];
        for (int k = 1; k < FA_WARPS; k++) s = fmin(s, r->d[k]);
        r->d[FA_WARPS] = s;
    }
    __syncthreads();
    return r->d[FA_WARPS];
}

__device__ __forceinline__ double block_max(double v, BlockRed* r) {
    v = warp_max(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) r->d[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = r->d[0];
        for (int k = 1; k < FA_WARPS; k++) s = fmax(s, r->d[k]);
        r->d[FA_WARPS] = s;
    }
    __syncthreads();
    return r->d[FA_WARPS];
}

// index of the FIRST minimum of key(i) over the caller's strided elements (np.argmin)
__device__ __forceinline__ int block_argmin_first(double key, int idx, BlockRed* r) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ok = __shfl_xor_sync(0xffffffffu, key, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ok < key || (ok == key && oi < idx)) { key = ok; idx = oi; }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { r->d[threadIdx.x >> 5] = key; r->i[threadIdx.x >> 5] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double k0 = r->d[0];
        int i0 = r->i[0];
        for (int k = 1; k < FA_WARPS; k++)
            if (r->d[k] < k0 || (r->d[k] == k0 && r->i[k] < i0)) { k0 = r->d[k]; i0 = r->i[k]; }
        r->i[FA_WARPS] = i0;
    }
    __syncthreads();
    return r->i[FA_WARPS];
}

// peak work arrays of one (frame, axis) in global scratch: 5 double arrays + 5 int arrays of `cap` entries after the profile arrays
__device__ __forceinline__ void peak_work_at(PeakWork& w, double* p, int cap, int* s_small) {
    w.cap = cap;
    w.prom = p; w.width_height = p + cap; w.lip = p + 2 * (size_t)cap; w.rip = p + 3 * (size_t)cap; w.skey = p + 4 * (size_t)cap;
    int* q = reinterpret_cast<int*>(p + 5 * (size_t)cap);
    w.idx = q; w.lbase = q + cap; w.rbase = q + 2 * (size_t)cap; w.flag = q + 3 * (size_t)cap; w.sidx = q + 4 * (size_t)cap;
    w.s_small = s_small;
}

// ------------------------------------------------------------------------------------------------ SingleProfile engine
struct Sp {
    // geometry of the (interpolated) profile: x_indices = np.linspace(start, stop, n)
    int n, n0;
    double start, stop, step;
    double dpmm;              // the detector's dpmm (indices are reported in detector pixels)
    int edge;                 // 0 FWHM, 1 inflection derivative, 2 edges supplied by the caller (Hill fits made on the host)
    double ov_l, ov_r;        // edge == 2: the supplied left / right edge positions
    const double* xg = nullptr;   // explicit (possibly uneven) abscissae of a pre-sampled profile, else the analytic linspace
    int centering;            // 2 geometric centre, else beam centre
    double smoothing;
    const double* gw;         // gaussian weights (2 * lw + 1) for this profile length, may be null
    int lw;
    double* v;                // values (n)
    double* t1;               // scratch (n)
    double* t2;               // scratch (n)
    PeakWork* w;
    BlockRed* red;
    double* bc;               // >= 8 doubles of shared broadcast space
    int* status;
};

__device__ __forceinline__ double sp_x(const Sp& s, int i) {
    if (s.xg) return s.xg[i];
    return i == s.n - 1 && s.n > 1 ? s.stop : (double)i * s.step + s.start;
}

// np.interp(loc, arange(n), x_indices)  (interp1d(range(n), x_indices): interior only)
__device__ __forceinline__ double sp_x_orig(const Sp& s, double loc) {
    if (loc >= (double)(s.n - 1)) return sp_x(s, s.n - 1);
    int j = (int)floor(loc);
    if (j < 0) j = 0;
    const double xj = (double)j;
    if (loc == xj) return sp_x(s, j);
    const double slope = (sp_x(s, j + 1) - sp_x(s, j)) / ((double)(j + 1) - xj);
    return slope * (loc - xj) + sp_x(s, j);
}

// np.searchsorted(x_indices, q, side) on the analytic grid
__device__ __forceinline__ int sp_searchsorted(const Sp& s, double q, bool right) {
    int lo = 0, hi = s.n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const double x = sp_x(s, mid);
        if (right ? (x <= q) : (x < q)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// interp1d(x_indices, values, kind='linear', fill_value='extrapolate')(q)
__device__ __forceinline__ double sp_y_at(const Sp& s, const double* __restrict__ v, double q) {
    int idx = sp_searchsorted(s, q, false);
    idx = min(max(idx, 1), s.n - 1);
    const int lo = idx - 1;
    const double xl = sp_x(s, lo), xh = sp_x(s, idx);
    const double slope = (v[idx] - v[lo]) / (xh - xl);
    return slope * (q - xl) + v[lo];
}

// find_peaks(values, fwxm_height=x/100, max_number=1): left / right interpolated positions of the most prominent peak
__device__ inline bool sp_fwxm(const Sp& s, double x_percent, double* left, double* right) {
    PeakArgs a;
    a.hmin = -INFINITY;
    a.distance = 1;
    a.pmin = -1.0;
    a.wmin = 0.0;
    a.rel_height = 1.0 - x_percent / 100;
    a.max_number = 1;
    a.sort_by_height = 0;
    const int np = block_find_peaks(s.v, s.n, a, *s.w);
    __syncthreads();
    if (np < 1) return false;
    const double l = s.w->lip[0], r = s.w->rip[0];
    __syncthreads();
    *left = sp_x_orig(s, l);
    *right = sp_x_orig(s, r);
    return true;
}

// inflection_data(): left-most peak / right-most valley of the gradient of the gaussian-smoothed profile
__device__ inline bool sp_inflection(const Sp& s, double* left, double* right) {
    const int n = s.n, tid = threadIdx.x;
    const double* __restrict__ gw = s.gw;
    const int lw = s.lw;
    auto at = [&](int idx) -> double {
        while (idx < 0 || idx >= n) {
            if (idx < 0) idx = -idx - 1;
            if (idx >= n) idx = 2 * n - 1 - idx;
        }
        return s.v[idx];
    };
    for (int l = tid; l < n; l += FA_THREADS) {
        double tmp;
        if (l - lw >= 0 && l + lw < n) {      // interior: every tap is inside the profile (same operands and order, no reflection tests)
            const double* __restrict__ q = s.v + l;
            tmp = q[0] * gw[lw];
            for (int ll = -lw; ll < 0; ll++) tmp += (q[ll] + q[-ll]) * gw[ll + lw];
        } else {
            tmp = at(l) * gw[lw];
            for (int ll = -lw; ll < 0; ll++) tmp += (at(l + ll) + at(l - ll)) * gw[ll + lw];
        }
        s.t1[l] = tmp;
    }
    __syncthreads();
    // np.gradient (edge_order 1): (f[i+1] - f[i-1]) / 2, one-sided at the ends
    double dmin = INFINITY, dmax = -INFINITY;
    for (int i = tid; i < n; i += FA_THREADS) {
        double g;
        if (n < 2) g = 0.0;
        else if (i == 0) g = (s.t1[1] - s.t1[0]) / 1.0;
        else if (i == n - 1) g = (s.t1[n - 1] - s.t1[n - 2]) / 1.0;
        else g = (s.t1[i + 1] - s.t1[i - 1]) / 2.0;
        s.t2[i] = g;
        dmin = fmin(dmin, g);
        dmax = fmax(dmax, g);
    }
    dmin = block_min(dmin, s.red);
    dmax = block_max(dmax, s.red);
    PeakArgs a;
    a.distance = max((int)(0.05 * (double)n), 1);
    a.pmin = -1.0;
    a.wmin = 0.0;
    a.rel_height = 1.0 - 0.5;
    a.max_number = 0;
    a.sort_by_height = 0;
    // MultiProfile(d1).find_peaks(threshold=0.8): threshold = min + 0.8 * (max - min)
    a.hmin = dmin + 0.8 * (dmax - dmin);
    int np = block_find_peaks(s.t2, n, a, *s.w);
    __syncthreads();
    if (np < 1) return false;
    const int pk = s.w->idx[0];
    __syncthreads();
    // find_valleys: the same on -d1 (min(-d1) = -max(d1))
    for (int i = tid; i < n; i += FA_THREADS) s.t1[i] = -s.t2[i];
    __syncthreads();
    a.hmin = -dmax + 0.8 * (-dmin - -dmax);
    np = block_find_peaks(s.t1, n, a, *s.w);
    __syncthreads();
    if (np < 1) return false;
    const int vl = s.w->idx[np - 1];
    __syncthreads();
    *left = sp_x_orig(s, (double)pk);
    *right = sp_x_orig(s, (double)vl);
    return true;
}

struct SpBeam { double idx, val_at_rounded; bool ok; double infl_l, infl_r; };

// beam_center() (core/profile.py:1381-1398)
__device__ inline SpBeam sp_beam_center(const Sp& s) {
    SpBeam b;
    b.infl_l = b.infl_r = 0.0;
    if (s.edge == 2) {
        b.ok = true;
        b.infl_l = s.ov_l;
        b.infl_r = s.ov_r;
        b.idx = s.ov_l + (s.ov_r - s.ov_l) / 2;
    } else if (s.edge == 0) {
        double l, r;
        b.ok = sp_fwxm(s, 50.0, &l, &r);
        if (!b.ok) { b.idx = 0; b.val_at_rounded = 1.0; return b; }
        b.idx = (r - l) / 2 + l;
    } else {
        double l, r;
        b.ok = sp_inflection(s, &l, &r);
        if (!b.ok) { b.idx = 0; b.val_at_rounded = 1.0; return b; }
        b.infl_l = l;
        b.infl_r = r;
        b.idx = l + (r - l) / 2;
    }
    b.val_at_rounded = sp_y_at(s, s.v, rint(b.idx));
    return b;
}

__device__ __forceinline__ double sp_geom_index(const Sp& s) { return sp_x_orig(s, (double)(s.n - 1) / 2.0); }

// SingleProfile.__init__: interpolation (NONE / LINEAR), ground, normalisation.  raw: n0 values.  Returns false on failure.
// interpolate: 0 none, 1 linear, 2 = `raw` is already sampled on np.linspace(xs, xe, n0) (host-side cubic interpolation / custom x_values)
__device__ inline bool sp_build(Sp& s, const double* __restrict__ raw, int n0, int interpolate, bool use_dpmm, double res_or_factor,
                                bool ground, int norm, double xs = 0.0, double xe = 0.0) {
    const int tid = threadIdx.x;
    s.n0 = n0;
    if (interpolate == 2) {
        s.n = n0;
        s.start = xs;
        s.stop = xe;
        s.step = (xe - xs) / (double)(n0 - 1);
        for (int i = tid; i < n0; i += FA_THREADS) s.v[i] = raw[i];
    } else if (!interpolate) {
        s.n = n0;
        s.start = 0.0;
        s.stop = (double)(n0 - 1);
        s.step = 1.0;
        for (int i = tid; i < n0; i += FA_THREADS) s.v[i] = raw[i];
    } else {
        // samples = int(round(len / (dpmm * resolution)))  or  int(round(len * factor))
        const double sm = use_dpmm ? (double)n0 / (s.dpmm * res_or_factor) : (double)n0 * res_or_factor;
        const int samples = (int)rint(sm);
        const double rf = (double)samples / (double)n0;
        const double offset = 0.5 - 1 / (2 * rf);
        s.n = samples;
        s.start = 0.0 - offset;
        s.stop = (double)(n0 - 1) + offset;
        s.step = (s.stop - s.start) / (double)(samples - 1);       // np.linspace
        for (int i = tid; i < samples; i += FA_THREADS) {
            const double xq = sp_x(s, i);
            // interp1d over integer knots 0..n0-1: searchsorted(x, xq) (side left), clipped to [1, n0 - 1]
            int idx = (int)ceil(xq);
            idx = min(max(idx, 1), n0 - 1);
            const int lo = idx - 1;
            const double slope = (raw[idx] - raw[lo]) / ((double)idx - (double)lo);
            s.v[i] = slope * (xq - (double)lo) + raw[lo];
        }
    }
    __syncthreads();
    const int n = s.n;
    if (ground) {
        double m = INFINITY;
        for (int i = tid; i < n; i += FA_THREADS) m = fmin(m, s.v[i]);
        m = block_min(m, s.red);
        for (int i = tid; i < n; i += FA_THREADS) s.v[i] -= m;
        __syncthreads();
    }
    double div = 1.0;
    bool ok = true;
    if (norm == 3) {                 // MAX
        double m = -INFINITY;
        for (int i = tid; i < n; i += FA_THREADS) m = fmax(m, s.v[i]);
        div = block_max(m, s.red);
    } else if (norm == 1) {          // GEOMETRIC_CENTER: geometric_center_value (core/array_utils.py:46-60)
        div = (n % 2 == 0) ? (s.v[n / 2] + s.v[n / 2 - 1]) / 2.0 : s.v[(n - 1) / 2];
    } else if (norm == 2) {          // BEAM_CENTER
        const SpBeam b = sp_beam_center(s);
        ok = b.ok;
        div = b.val_at_rounded;
    }
    __syncthreads();
    if (norm != 0 && ok) {
        for (int i = tid; i < n; i += FA_THREADS) s.v[i] = s.v[i] / div;
        __syncthreads();
    }
    return ok;
}

// _sample_points_in_physical_window -> [start, stop) on the sample grid
__device__ inline void sp_window(const Sp& s, double a, double b, int* start_out, int* stop_out) {
    const double lower = fmin(a, b), upper = fmax(a, b);
    int start = sp_searchsorted(s, lower, false);
    int stop = sp_searchsorted(s, upper, true);
    if (stop - start < 3) {
        // nearest samples: x_indices is increasing, the first minimum of |x - q| is next to searchsorted(q)
        auto nearest = [&](double q) {
            int j = sp_searchsorted(s, q, false);
            int best = min(max(j, 0), s.n - 1);
            double bd = fabs(sp_x(s, best) - q);
            for (int k = max(j - 2, 0); k <= min(j + 1, s.n - 1); k++) {
                const double d = fabs(sp_x(s, k) - q);
                if (d < bd || (d == bd && k < best)) { bd = d; best = k; }
            }
            return best;
        };
        const int li = nearest(lower), ri = nearest(upper);
        start = min(li, ri);
        stop = max(li, ri) + 1;
        if (stop - start < 3) {
            const int c = nearest((lower + upper) / 2);
            start = max(0, c - 1);
            stop = min(s.n, start + 3);
            start = max(0, stop - 3);
        }
    }
    *start_out = start;
    *stop_out = stop;
}

// scipy.stats.linregress slope of (x_indices[i], y_at(x_indices[i])) over [start, stop)
__device__ inline double sp_window_slope(const Sp& s, int start, int stop, double* intercept = nullptr) {
    const int tid = threadIdx.x, m = stop - start;
    double sx = 0, sy = 0;
    for (int i = start + tid; i < stop; i += FA_THREADS) { sx += sp_x(s, i); sy += sp_y_at(s, s.v, sp_x(s, i)); }
    const double xm = block_sum(sx, s.red) / m, ym = block_sum(sy, s.red) / m;
    double sxx = 0, sxy = 0;
    for (int i = start + tid; i < stop; i += FA_THREADS) {
        const double dx = sp_x(s, i) - xm;
        sxx += dx * dx;
        sxy += dx * (sp_y_at(s, s.v, sp_x(s, i)) - ym);
    }
    const double ssxm = block_sum(sxx, s.red) / m, ssxym = block_sum(sxy, s.red) / m;
    const double slope = ssxym / ssxm;
    if (intercept) *intercept = ym - slope * xm;
    return slope;
}

struct SpField {
    bool ok;
    double width, beam_center, cax, beam_center_val, left, right, left_slope, right_slope, top;
    double inner_left, inner_right, left_intercept, right_intercept, top_val, top_params[3];
    int fv_n;               // number of "field values" left in s.t1
};

// field_data(in_field_ratio, slope_exclusion_ratio); leaves the "field values" in s.t1[0 .. fv_n)
__device__ inline SpField sp_field_data(const Sp& s, double ifr, double ser) {
    SpField f;
    f.ok = false;
    f.fv_n = 0;
    f.width = f.beam_center = f.cax = f.beam_center_val = f.left = f.right = f.left_slope = f.right_slope = f.top = 0.0;
    f.inner_left = f.inner_right = f.left_intercept = f.right_intercept = f.top_val = 0.0;
    f.top_params[0] = f.top_params[1] = f.top_params[2] = 0.0;
    const int tid = threadIdx.x;
    double full_width;
    if (s.edge == 0) {
        double l, r;
        if (!sp_fwxm(s, 50.0, &l, &r)) return f;
        f.beam_center = (r - l) / 2 + l;
        full_width = r - l;
    } else {
        const SpBeam b = sp_beam_center(s);
        if (!b.ok) return f;
        f.beam_center = b.idx;
        full_width = b.infl_r - b.infl_l;
    }
    f.cax = sp_geom_index(s);
    const double center = s.centering == 2 ? f.cax : f.beam_center;
    const double fl = center - ifr * full_width / 2;
    const double fr = center + ifr * full_width / 2;
    const double fw = fr - fl;
    const double il = center - ser * fw / 2;
    const double ir = center + ser * fw / 2;
    int a0, a1;
    sp_window(s, fl, il, &a0, &a1);
    f.left_slope = sp_window_slope(s, a0, a1, &f.left_intercept);
    sp_window(s, ir, fr, &a0, &a1);
    f.right_slope = sp_window_slope(s, a0, a1, &f.right_intercept);
    f.inner_left = il;
    f.inner_right = ir;
    // top: np.polyfit(top_x, top_y, 2) as least squares on u = (x - mean) / max|x - mean|, vertex clipped to the window
    sp_window(s, il, ir, &a0, &a1);
    {
        const int m = a1 - a0;
        double sx = 0;
        for (int i = a0 + tid; i < a1; i += FA_THREADS) sx += sp_x(s, i);
        const double xm = block_sum(sx, s.red) / m;
        const double sc0 = fmax(fabs(sp_x(s, a0) - xm), fabs(sp_x(s, a1 - 1) - xm));
        const double sc = sc0 > 0 ? sc0 : 1.0;
        double s1 = 0, s2 = 0, s3 = 0, s4 = 0, t0 = 0, t1 = 0, t2 = 0;
        for (int i = a0 + tid; i < a1; i += FA_THREADS) {
            const double u = (sp_x(s, i) - xm) / sc, y = sp_y_at(s, s.v, sp_x(s, i));
            const double u2 = u * u;
            s1 += u; s2 += u2; s3 += u2 * u; s4 += u2 * u2;
            t0 += y; t1 += u * y; t2 += u2 * y;
        }
        s1 = block_sum(s1, s.red); s2 = block_sum(s2, s.red); s3 = block_sum(s3, s.red); s4 = block_sum(s4, s.red);
        t0 = block_sum(t0, s.red); t1 = block_sum(t1, s.red); t2 = block_sum(t2, s.red);
        // normal equations [[s4 s3 s2][s3 s2 s1][s2 s1 m]] (c2 c1 c0)^T = (t2 t1 t0)^T, Cramer
        const double M = (double)m;
        const double det = s4 * (s2 * M - s1 * s1) - s3 * (s3 * M - s1 * s2) + s2 * (s3 * s1 - s2 * s2);
        const double c2 = (t2 * (s2 * M - s1 * s1) - s3 * (t1 * M - s1 * t0) + s2 * (t1 * s1 - s2 * t0)) / det;
        const double c1 = (s4 * (t1 * M - t0 * s1) - t2 * (s3 * M - s1 * s2) + s2 * (s3 * t0 - s2 * t1)) / det;
        const double c0 = (s4 * (s2 * t0 - s1 * t1) - s3 * (s3 * t0 - t1 * s2) + t2 * (s3 * s1 - s2 * s2)) / det;
        const double lo_u = (sp_x(s, a0) - xm) / sc, hi_u = (sp_x(s, a1 - 1) - xm) / sc;
        double best_u = lo_u, best_v = c2 * lo_u * lo_u + c1 * lo_u + c0;
        const double hv = c2 * hi_u * hi_u + c1 * hi_u + c0;
        if (hv > best_v) { best_v = hv; best_u = hi_u; }
        if (c2 != 0) {
            const double vx = -c1 / (2 * c2);
            if (vx >= lo_u && vx <= hi_u) {
                const double vv = c2 * vx * vx + c1 * vx + c0;
                if (vv > best_v) { best_v = vv; best_u = vx; }
            }
        }
        // The reference does not take the vertex: it runs scipy.optimize.minimize(-parabola, x0 = middle of the window, bounds =
        // window), i.e. L-BFGS-B with a finite-difference gradient (core/profile.py:1533-1542).  Field tops are nearly flat in index
        // units (curvature ~1e-6 / px^2), so the run ends in one of L-BFGS-B's first two tests, restated here for a 1-D parabola:
        //   projected gradient at x0 <= pgtol (1e-5)                                   -> x0
        //   x1 = x0 - g0 (Cauchy step of the unit-Hessian model; boxed problem: step 1), then
        //   projected gradient at x1 <= pgtol, or f0 - f1 <= ftol max(|f0|, |f1|, 1)   -> x1      (ftol = 2.22e-9)
        //   otherwise the iteration converges to the constrained minimum               -> vertex / better bound (above)
        {
            const double lo_x = sp_x(s, a0), hi_x = sp_x(s, a1 - 1);
            auto par = [&](double x) { const double u = (x - xm) / sc; return c2 * u * u + c1 * u + c0; };
            auto grad = [&](double x) { return -(2 * c2 * ((x - xm) / sc) + c1) / sc; };
            auto proj = [&](double x, double g) { return g < 0 ? fmax(x - hi_x, g) : fmin(x - lo_x, g); };
            const double x0 = lo_x + fabs(hi_x - lo_x) / 2;
            const double g0 = grad(x0);
            double top = best_u * sc + xm;
            if (fabs(proj(x0, g0)) <= 1e-5) {
                top = x0;
            } else {
                const double x1 = fmin(fmax(x0 - g0, lo_x), hi_x);
                const double f0 = -par(x0), f1 = -par(x1);
                if (fabs(proj(x1, grad(x1))) <= 1e-5 || f0 - f1 <= 2.220446049250313e-09 * fmax(fmax(fabs(f0), fabs(f1)), 1.0)) top = x1;
            }
            f.top = top;
            f.top_val = par(top);
        }
        // coefficients of np.polyfit in the abscissa itself: u = (x - xm) / sc
        f.top_params[0] = c2 / (sc * sc);
        f.top_params[1] = c1 / sc - 2 * c2 * xm / (sc * sc);
        f.top_params[2] = c0 - c1 * xm / sc + c2 * xm * xm / (sc * sc);
    }
    // field values: y_at(x_indices_shifted[imin .. imax]) with the pixel-offset shift (core/profile.py:1563-1574)
    const double off = center - rint(center);
    double kmin = INFINITY, kmax = INFINITY;
    int imn = 0x7fffffff, imx = 0x7fffffff;
    for (int i = tid; i < s.n; i += FA_THREADS) {
        const double xs = sp_x(s, i) + off;
        const double d0 = fabs(xs - fl), d1 = fabs(xs - fr);
        if (d0 < kmin) { kmin = d0; imn = i; }
        if (d1 < kmax) { kmax = d1; imx = i; }
    }
    const int x_index_min = block_argmin_first(kmin, imn, s.red);
    const int x_index_max = block_argmin_first(kmax, imx, s.red);
    const int nfv = x_index_max >= x_index_min ? x_index_max - x_index_min + 1 : 0;
    for (int i = tid; i < nfv; i += FA_THREADS) s.t1[i] = sp_y_at(s, s.v, sp_x(s, x_index_min + i) + off);
    __syncthreads();
    f.fv_n = nfv;
    f.width = fw;
    f.left = fl;
    f.right = fr;
    f.beam_center_val = sp_y_at(s, s.v, rint(f.beam_center));
    f.ok = true;
    return f;
}

// ------------------------------------------------------------------------------------------------ kernels
// CTA per (frame, axis): axis 0 = profile of the row sums (np.sum(array, 1), decides horiz_position), axis 1 = column sums.
__global__ void __launch_bounds__(FA_THREADS)
k_field_center(const FieldConst* __restrict__ cc, const FrameStats* __restrict__ stats, const uint32_t* __restrict__ rowsum,
               const uint32_t* __restrict__ colsum, FieldFrame* ff, double* __restrict__ work, epid_field_result* __restrict__ res) {
    __shared__ int s_small[FA_THREADS + 8];
    __shared__ BlockRed s_red;
    __shared__ double s_bc[8];
    __shared__ int s_status;
    const FieldConst& c = *cc;
    const int fi = blockIdx.x, axis = blockIdx.y;
    const int tid = threadIdx.x;
    const int H = c.H, W = c.W;
    const FrameStats fs = stats[fi];
    FieldFrame& f = ff[fi];
    // check_inversion_by_histogram() with the default percentiles (5, 50, 95) (field_analysis.py:472, core/image.py:899-926)
    const int hist_inv = stats_hist_inverted(fs, c.p5.gamma, c.p50.gamma, c.p95.gamma);      // certified from counts or exact percentiles
    const int flip = hist_inv ^ (c.p.invert ? 1 : 0);
    if (tid == 0 && axis == 0) {
        f.mn = fs.mn;
        f.mx = fs.mx;
        f.flip = flip;
        f.hist_inverted = hist_inv;
        epid_field_result& R = res[fi];
        if (fs.mn == fs.mx) R.status = EPID_FIELD_FLAT_IMAGE;      // results are zero-initialised (EPID_FIELD_OK)
        R.hist_inverted = hist_inv;
    }
    const int n0 = axis == 0 ? H : W;          // axis 0: vert_sum (one value per row)
    const int other = axis == 0 ? W : H;
    double pos = axis == 0 ? c.p.horiz_position : c.p.vert_position;
    if (c.p.centering != 0) {
        double* base = work + ((size_t)fi * 2 + axis) * c.stride;
        double* raw = base + 3 * (size_t)c.nmax;
        const uint32_t* src = axis == 0 ? rowsum + (size_t)fi * H : colsum + (size_t)fi * W;
        const double inv_const = (double)other * ((double)fs.mx + (double)fs.mn);
        for (int i = tid; i < n0; i += FA_THREADS) raw[i] = flip ? inv_const - (double)src[i] : (double)src[i];
        __syncthreads();
        PeakWork w;
        peak_work_at(w, base + 4 * (size_t)c.nmax, c.pcap, s_small);
        Sp s;
        s.dpmm = 0.0;
        s.edge = 0;
        s.centering = 1;
        s.smoothing = 0.0;
        s.gw = nullptr;
        s.lw = 0;
        s.v = base;
        s.t1 = base + c.nmax;
        s.t2 = base + 2 * (size_t)c.nmax;
        s.w = &w;
        s.red = &s_red;
        s.bc = s_bc;
        s.status = &s_status;
        // SingleProfile(sum) with its defaults: LINEAR x10, ground, BEAM_CENTER normalisation, FWHM edges
        bool ok = 10 * n0 <= c.nmax && sp_build(s, raw, n0, true, false, 10.0, true, 2);
        if (ok) {
            if (c.p.centering == 2) {
                pos = sp_geom_index(s) / (double)n0;
            } else {
                const SpBeam b = sp_beam_center(s);
                ok = b.ok;
                pos = b.idx / (double)n0;
            }
        }
        if (!ok && tid == 0) res[fi].status = EPID_FIELD_NO_EDGES;
    }
    if (tid == 0) {
        // _get_horiz_values / _get_vert_values (field_analysis.py:1069-1117)
        const double width = axis == 0 ? c.p.horiz_width : c.p.vert_width;
        int lo = (int)rint((double)n0 * pos - (double)n0 * width / 2);
        lo = max(lo, 0);
        int hi = (int)rint((double)n0 * pos + (double)n0 * width / 2) + 1;
        hi = min(hi, n0);
        f.pos[axis] = pos;
        f.lo[axis] = lo;
        f.hi[axis] = hi;
        epid_field_result& R = res[fi];
        if (axis == 0) { R.strip_rows[0] = lo; R.strip_rows[1] = hi; }
        else { R.strip_cols[0] = lo; R.strip_cols[1] = hi; }
    }
}

// CTA per (frame, axis): axis 0 = horizontal profile (mean over rows [lo, hi) for every column), axis 1 = vertical profile.
__global__ void __launch_bounds__(FA_THREADS)
k_field_strips(const FieldConst* __restrict__ cc, const FrameRef* __restrict__ frames, const FieldFrame* __restrict__ ff,
               double* __restrict__ work) {
    const FieldConst& c = *cc;
    const int fi = blockIdx.x, axis = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int H = c.H, W = c.W;
    const FrameRef frf = frames[fi];
    const FieldFrame f = ff[fi];
    double* raw = work + ((size_t)fi * 2 + axis) * c.stride + 3 * (size_t)c.nmax;
    const uint32_t sum_c = f.mx + f.mn;
    const int lo = f.lo[axis], hi = f.hi[axis];
    const int cnt = hi - lo;
    if (axis == 0) {
        // np.mean(array[bottom:top, :], 0): exact integer sum / count
        for (int x = tid; x < W; x += FA_THREADS) {
            unsigned long long acc = 0;
            for (int y = lo; y < hi; y++) {
                const uint32_t v = __ldg(frf.origin + (size_t)y * frf.pitch + x);
                acc += f.flip ? sum_c - v : v;
            }
            raw[x] = cnt > 0 ? (double)acc / (double)cnt : __longlong_as_double(0x7ff8000000000000LL);
        }
    } else {
        for (int y = wid; y < H; y += FA_WARPS) {
            unsigned long long acc = 0;
            for (int x = lo + lane; x < hi; x += 32) {
                const uint32_t v = __ldg(frf.origin + (size_t)y * frf.pitch + x);
                acc += f.flip ? sum_c - v : v;
            }
            acc = warp_sum(acc);
            if (lane == 0) raw[y] = cnt > 0 ? (double)acc / (double)cnt : __longlong_as_double(0x7ff8000000000000LL);
        }
    }
}

#ifndef EPID_FA_MIN_CTAS
#define EPID_FA_MIN_CTAS 2      // resident CTAs per SM k_field_profile is compiled for (3: 80 registers, ~0.9 KB of spill traffic; variants/)
#endif
__global__ void __launch_bounds__(FA_THREADS, EPID_FA_MIN_CTAS)
k_field_profile(const FieldConst* __restrict__ cc, const double* __restrict__ gw_h, const double* __restrict__ gw_v,
                double* __restrict__ work, epid_field_result* __restrict__ res) {
    __shared__ int s_small[FA_THREADS + 8];
    __shared__ BlockRed s_red;
    __shared__ double s_bc[8];
    __shared__ int s_status;
    const FieldConst& c = *cc;
    const int fi = blockIdx.x, axis = blockIdx.y;
    const int tid = threadIdx.x;
    epid_field_result& R = res[fi];
    if (R.status != EPID_FIELD_OK) return;
    const int n0 = axis == 0 ? c.W : c.H;
    double* base = work + ((size_t)fi * 2 + axis) * c.stride;
    const double* raw = base + 3 * (size_t)c.nmax;
    PeakWork w;
    peak_work_at(w, base + 4 * (size_t)c.nmax, c.pcap, s_small);
    Sp s;
    s.dpmm = c.p.dpmm;
    s.edge = c.p.edge;
    s.centering = 1;                      // FieldAnalysis does not forward `centering` to its SingleProfiles (field_analysis.py:528-562)
    s.smoothing = c.p.edge_smoothing_ratio;
    s.gw = axis == 0 ? gw_h : gw_v;
    s.lw = c.lw[axis];
    s.v = base;
    s.t1 = base + c.nmax;
    s.t2 = base + 2 * (size_t)c.nmax;
    s.w = &w;
    s.red = &s_red;
    s.bc = s_bc;
    s.status = &s_status;
    const bool interp = c.p.interpolation != 0;
    bool ok = sp_build(s, raw, n0, interp, true, c.p.interpolation_resolution_mm, c.p.ground != 0, c.p.normalization);
    if (ok && s.edge == 1 && s.n != c.n_expect[axis]) ok = false;      // the gaussian weights were made for another length
    double out[16];
    for (int k = 0; k < 16; k++) out[k] = 0.0;
    // ---- penumbra(lower, upper) (core/profile.py:1723-1907)
    if (ok) {
        const double lower = c.p.penumbra_lower, upper = c.p.penumbra_upper;
        double ll, lr, ul, ur, dummy;
        if (s.edge == 0) {
            ok = sp_fwxm(s, upper, &ul, &ur) && sp_fwxm(s, lower, &ll, &lr);
        } else {
            double il, ir;
            ok = sp_inflection(s, &il, &ir);
            if (ok) {
                const double vl = sp_y_at(s, s.v, il), vr = sp_y_at(s, s.v, ir);
                double vmax = -INFINITY;
                for (int i = tid; i < s.n; i += FA_THREADS) vmax = fmax(vmax, s.v[i]);
                vmax = block_max(vmax, s.red);
                const double lo_l = fmax(vl / vmax * lower / 50 * 100, 1.0), up_l = fmin(vl / vmax * upper / 50 * 100, 99.0);
                const double lo_r = fmax(vr / vmax * lower / 50 * 100, 1.0), up_r = fmin(vr / vmax * upper / 50 * 100, 99.0);
                ok = sp_fwxm(s, up_l, &ul, &dummy) && sp_fwxm(s, lo_l, &ll, &dummy) && sp_fwxm(s, up_r, &dummy, &ur) &&
                     sp_fwxm(s, lo_r, &dummy, &lr);
            }
        }
        if (ok) {
            out[0] = fabs(ul - ll) / s.dpmm;        // left penumbra width (exact) mm
            out[1] = fabs(ur - lr) / s.dpmm;        // right
        }
    }
    // ---- geometric / beam centre
    if (ok) {
        out[2] = sp_geom_index(s);
        const SpBeam b = sp_beam_center(s);
        ok = b.ok;
        out[3] = b.idx;
    }
    // ---- field_data(in_field_ratio=1.0): sizes and distances
    if (ok) {
        const SpField f1 = sp_field_data(s, 1.0, c.p.slope_exclusion_ratio);
        ok = f1.ok;
        if (ok) {
            out[4] = f1.width / s.dpmm;
            out[5] = fabs(f1.beam_center - f1.left) / s.dpmm;
            out[6] = fabs(f1.right - f1.beam_center) / s.dpmm;
            out[7] = fabs(f1.cax - f1.left) / s.dpmm;
            out[8] = fabs(f1.cax - f1.right) / s.dpmm;
        }
    }
    // ---- field_data(in_field_ratio): top, slopes, protocol
    if (ok) {
        const SpField f2 = sp_field_data(s, c.p.in_field_ratio, c.p.slope_exclusion_ratio);
        ok = f2.ok;
        if (ok) {
            out[9] = f2.top;
            out[10] = fabs(f2.top - f2.cax) / s.dpmm;
            out[11] = (f2.top - f2.beam_center) / s.dpmm;
            out[12] = f2.left_slope * s.dpmm * 100;
            out[13] = f2.right_slope * s.dpmm * 100;
            const int m = f2.fv_n;
            const double* fv = s.t1;
            const int proto = c.p.protocol;
            if (proto != 0 && m > 0) {
                // flatness: VARIAN / SIEMENS dose difference, ELEKTA dose ratio (field_analysis.py:37-85).  The ELEKTA ratio is
                // taken with the default slope_exclusion_ratio of field_calculation (0.2), which does not change the field values.
                double vmin = INFINITY, vmax = -INFINITY;
                for (int i = tid; i < m; i += FA_THREADS) { vmin = fmin(vmin, fv[i]); vmax = fmax(vmax, fv[i]); }
                vmin = block_min(vmin, s.red);
                vmax = block_max(vmax, s.red);
                out[15] = proto == 3 ? 100 * (vmax / vmin) : 100 * fabs(vmax - vmin) / (vmax + vmin);
                if (proto == 2) {
                    // symmetry_area (field_analysis.py:179-194)
                    double al = 0, ar = 0;
                    const int nl = m / 2, r0 = (m + 1) / 2;
                    for (int i = tid; i < nl; i += FA_THREADS) al += fv[i];
                    for (int i = r0 + tid; i < m; i += FA_THREADS) ar += fv[i];
                    al = block_sum(al, s.red);
                    ar = block_sum(ar, s.red);
                    out[14] = 100 * (al - ar) / (al + ar);
                } else {
                    // point difference (VARIAN) / PDQ IEC (ELEKTA): value of the first maximum of |sym| (np.argmax)
                    double best = -INFINITY;
                    int bi = 0x7fffffff;
                    for (int i = tid; i < m; i += FA_THREADS) {
                        const double lt = fv[i], rt = fv[m - 1 - i];
                        double sym;
                        if (proto == 1) {
                            sym = 100 * (lt - rt) / f2.beam_center_val;
                        } else {
                            const double s1 = lt / rt, s2 = rt / lt;
                            const double sg = fabs(s1) > fabs(s2) ? (double)((s1 > 0) - (s1 < 0)) : (double)((s2 > 0) - (s2 < 0));
                            sym = fmax(fabs(s1), fabs(s2)) * sg;
                        }
                        s.t2[i] = sym;
                        if (fabs(sym) > best) { best = fabs(sym); bi = i; }
                    }
                    const int arg = block_argmin_first(-best, bi, s.red);
                    out[14] = s.t2[arg];
                }
            }
        }
    }
    if (tid == 0) {
        if (!ok) { R.status = EPID_FIELD_NO_EDGES; return; }
        R.profile_len[axis] = s.n;
        if (axis == 0) {
            R.left_penumbra_mm = out[0]; R.right_penumbra_mm = out[1];
            R.geometric_center_index_x_y[0] = out[2]; R.beam_center_index_x_y[0] = out[3];
            R.field_size_horizontal_mm = out[4];
            R.beam_center_to_left_mm = out[5]; R.beam_center_to_right_mm = out[6];
            R.cax_to_left_mm = out[7]; R.cax_to_right_mm = out[8];
            R.top_position_index_x_y[0] = out[9];
            R.top_horizontal_distance_from_cax_mm = out[10];
            R.top_horizontal_distance_from_beam_center_mm = out[11];
            R.left_slope_percent_mm = out[12]; R.right_slope_percent_mm = out[13];
            R.symmetry_horizontal = out[14]; R.flatness_horizontal = out[15];
        } else {
            R.top_penumbra_mm = out[0]; R.bottom_penumbra_mm = out[1];
            R.geometric_center_index_x_y[1] = out[2]; R.beam_center_index_x_y[1] = out[3];
            R.field_size_vertical_mm = out[4];
            R.beam_center_to_top_mm = out[5]; R.beam_center_to_bottom_mm = out[6];
            R.cax_to_top_mm = out[7]; R.cax_to_bottom_mm = out[8];
            R.top_position_index_x_y[1] = out[9];
            R.top_vertical_distance_from_cax_mm = out[10];
            R.top_vertical_distance_from_beam_center_mm = out[11];
            R.top_slope_percent_mm = out[12]; R.bottom_slope_percent_mm = out[13];
            R.symmetry_vertical = out[14]; R.flatness_vertical = out[15];
        }
    }
}

// ------------------------------------------------------------------------------------------------ SingleProfile (one profile)
// SingleProfile(values, dpmm, ...) and its query methods for ONE host profile (core/profile.py:1125-1937): the same engine as
// k_field_profile, every query evaluated in one launch.
__global__ void __launch_bounds__(FA_THREADS)
k_single_profile(const epid_sp_params p, const double* __restrict__ raw, const double* __restrict__ xg, int n0, int nmax, int pcap, const double* __restrict__ gw, int lw,
                 int n_expect, double fwxm_x, double pen_lower, double pen_upper, double ifr, double ser, double* __restrict__ work,
                 epid_sp_result* __restrict__ out, double* __restrict__ values_out, double* __restrict__ fv_out) {
    __shared__ int s_small[FA_THREADS + 8];
    __shared__ BlockRed s_red;
    __shared__ double s_bc[8];
    __shared__ int s_status;
    const int tid = threadIdx.x;
    PeakWork w;
    peak_work_at(w, work + 3 * (size_t)nmax, pcap, s_small);
    Sp s;
    s.dpmm = p.dpmm;
    s.edge = p.edge;
    s.ov_l = p.edge_left;
    s.ov_r = p.edge_right;
    s.xg = p.interpolation == 2 ? xg : nullptr;
    s.centering = p.centering;
    s.smoothing = p.edge_smoothing_ratio;
    s.gw = gw;
    s.lw = lw;
    s.v = work;
    s.t1 = work + nmax;
    s.t2 = work + 2 * (size_t)nmax;
    s.w = &w;
    s.red = &s_red;
    s.bc = s_bc;
    s.status = &s_status;
    epid_sp_result R;
    memset(&R, 0, sizeof(R));
    const bool use_dpmm = p.dpmm > 0;
    bool ok = sp_build(s, raw, n0, p.interpolation, use_dpmm, use_dpmm ? p.interpolation_resolution_mm : p.interpolation_factor,
                       p.ground != 0, p.normalization, p.x_start, p.x_stop);
    if (ok && s.edge == 1 && s.n != n_expect) ok = false;
    R.status = ok ? 0 : 1;
    R.n = s.n;
    R.x_start = s.start;
    R.x_stop = s.stop;
    if (ok) {
        for (int i = tid; i < s.n; i += FA_THREADS) values_out[i] = s.v[i];
        double vmax = -INFINITY;
        for (int i = tid; i < s.n; i += FA_THREADS) vmax = fmax(vmax, s.v[i]);
        R.values_max = block_max(vmax, s.red);
        R.geometric_center_index = sp_geom_index(s);
        R.geometric_center_value = (s.n % 2 == 0) ? (s.v[s.n / 2] + s.v[s.n / 2 - 1]) / 2.0 : s.v[(s.n - 1) / 2];
        // fwxm_data(x)
        double l, r;
        if (sp_fwxm(s, fwxm_x, &l, &r)) {
            R.fwxm_ok = 1;
            R.fwxm_left = l;
            R.fwxm_right = r;
            const double c = (r - l) / 2 + l;
            R.fwxm_center_value_at_rounded = sp_y_at(s, s.v, rint(c));
            R.fwxm_left_value_at_rounded = sp_y_at(s, s.v, rint(l));
            R.fwxm_right_value_at_rounded = sp_y_at(s, s.v, rint(r));
        }
        // inflection_data()
        if (s.edge == 1) {
            double il, ir;
            if (sp_inflection(s, &il, &ir)) {
                R.infl_ok = 1;
                R.infl_left = il;
                R.infl_right = ir;
                R.infl_left_value_exact = sp_y_at(s, s.v, il);
                R.infl_right_value_exact = sp_y_at(s, s.v, ir);
                R.infl_left_value_rounded = sp_y_at(s, s.v, rint(il));
                R.infl_right_value_rounded = sp_y_at(s, s.v, rint(ir));
            }
        } else if (s.edge == 2) {
            R.infl_ok = 1;
            R.infl_left = s.ov_l;
            R.infl_right = s.ov_r;
            R.infl_left_value_exact = sp_y_at(s, s.v, s.ov_l);
            R.infl_right_value_exact = sp_y_at(s, s.v, s.ov_r);
            R.infl_left_value_rounded = sp_y_at(s, s.v, rint(s.ov_l));
            R.infl_right_value_rounded = sp_y_at(s, s.v, rint(s.ov_r));
        }
        // beam_center()
        const SpBeam b = sp_beam_center(s);
        if (b.ok) { R.beam_ok = 1; R.beam_center_index = b.idx; R.beam_center_value_at_rounded = b.val_at_rounded; }
        // penumbra(lower, upper)
        {
            double ll = 0, lr = 0, ul = 0, ur = 0, dummy;
            bool pk;
            if (s.edge == 0) {
                pk = sp_fwxm(s, pen_upper, &ul, &ur) && sp_fwxm(s, pen_lower, &ll, &lr);
            } else if (s.edge == 2) {
                pk = false;                 // Hill penumbra: closed form of the fitted parameters, evaluated by the caller
            } else {
                pk = R.infl_ok != 0;
                if (pk) {
                    const double lo_l = fmax(R.infl_left_value_exact / R.values_max * pen_lower / 50 * 100, 1.0);
                    const double up_l = fmin(R.infl_left_value_exact / R.values_max * pen_upper / 50 * 100, 99.0);
                    const double lo_r = fmax(R.infl_right_value_exact / R.values_max * pen_lower / 50 * 100, 1.0);
                    const double up_r = fmin(R.infl_right_value_exact / R.values_max * pen_upper / 50 * 100, 99.0);
                    pk = sp_fwxm(s, up_l, &ul, &dummy) && sp_fwxm(s, lo_l, &ll, &dummy) && sp_fwxm(s, up_r, &dummy, &ur) && sp_fwxm(s, lo_r, &dummy, &lr);
                }
            }
            if (pk) { R.pen_ok = 1; R.pen_left_lower = ll; R.pen_left_upper = ul; R.pen_right_lower = lr; R.pen_right_upper = ur; }
        }
        // field_data(in_field_ratio, slope_exclusion_ratio)
        if (ser < ifr) {
            const SpField f = sp_field_data(s, ifr, ser);
            if (f.ok) {
                R.fd_ok = 1;
                R.fd_width = f.width; R.fd_beam_center = f.beam_center; R.fd_cax = f.cax; R.fd_left = f.left; R.fd_right = f.right;
                R.fd_inner_left = f.inner_left; R.fd_inner_right = f.inner_right;
                R.fd_left_slope = f.left_slope; R.fd_left_intercept = f.left_intercept;
                R.fd_right_slope = f.right_slope; R.fd_right_intercept = f.right_intercept;
                R.fd_top_index = f.top; R.fd_top_value = f.top_val;
                R.fd_top_params[0] = f.top_params[0]; R.fd_top_params[1] = f.top_params[1]; R.fd_top_params[2] = f.top_params[2];
                R.fd_beam_center_value = f.beam_center_val;
                R.fd_cax_value = sp_y_at(s, s.v, rint(f.cax));
                R.fd_left_value = sp_y_at(s, s.v, rint(f.left));
                R.fd_right_value = sp_y_at(s, s.v, rint(f.right));
                R.fd_field_values_n = f.fv_n;
                for (int i = tid; i < f.fv_n; i += FA_THREADS) fv_out[i] = s.t1[i];
            }
        }
    }
    if (tid == 0) *out = R;
}

}  // namespace epid

using namespace epid;

extern "C" int32_t epid_field_profile_len(int32_t n0, double dpmm, int32_t interpolation, double resolution_mm) {
    if (!interpolation) return n0;
    return (int32_t)rint((double)n0 / (dpmm * resolution_mm));
}

extern "C" int32_t epid_field_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_field_params* p, const double* gauss_h,
                                      int32_t lw_h, const double* gauss_v, int32_t lw_v, epid_field_result* results) {
    EPID_REQUIRE(ctx && frames && p && results, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(frames->dtype == EPID_U16, EPID_ERR_UNSUPPORTED, "field analysis frames must be uint16");
    EPID_REQUIRE(p->dpmm > 0, EPID_ERR_INVALID, "dpmm must be positive");
    EPID_REQUIRE(p->slope_exclusion_ratio < p->in_field_ratio, EPID_ERR_INVALID, "The exclusion region must be smaller than the field ratio");
    EPID_REQUIRE(p->slope_exclusion_ratio < 1.0, EPID_ERR_INVALID, "The exclusion region must be smaller than the field ratio");
    EPID_REQUIRE(p->penumbra_lower <= p->penumbra_upper, EPID_ERR_INVALID, "Upper penumbra value must be larger than the lower penumbra value");
    EPID_REQUIRE(p->edge == 0 || (gauss_h && gauss_v), EPID_ERR_INVALID, "gaussian weights missing");
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = frames->n, H = frames->h, W = frames->w;
    FieldConst hc;
    memset(&hc, 0, sizeof(hc));
    hc.p = *p;
    hc.H = H;
    hc.W = W;
    hc.p5 = pct_plan(H * W, 5.0);
    hc.p50 = pct_plan(H * W, 50.0);
    hc.p95 = pct_plan(H * W, 95.0);
    hc.n_expect[0] = epid_field_profile_len(W, p->dpmm, p->interpolation, p->interpolation_resolution_mm);
    hc.n_expect[1] = epid_field_profile_len(H, p->dpmm, p->interpolation, p->interpolation_resolution_mm);
    int nmax = 10 * (H > W ? H : W);
    if (hc.n_expect[0] > nmax) nmax = hc.n_expect[0];
    if (hc.n_expect[1] > nmax) nmax = hc.n_expect[1];
    hc.nmax = nmax + 16;
    hc.pcap = 1;
    while (hc.pcap < hc.nmax / 2 + 8) hc.pcap <<= 1;
    hc.stride = 4 * (size_t)hc.nmax + 8 * (size_t)hc.pcap;
    hc.lw[0] = lw_h;
    hc.lw[1] = lw_v;
    EPID_REQUIRE(hc.n_expect[0] >= 8 && hc.n_expect[1] >= 8, EPID_ERR_UNSUPPORTED, "profile too short");
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    const size_t o_cst = sz(sizeof(FieldConst)), o_rf = sz(sizeof(FrameRef) * n), o_st = sz(sizeof(FrameStats) * n);
    const size_t o_rs = sz(sizeof(uint32_t) * (size_t)n * H), o_cs = sz(sizeof(uint32_t) * (size_t)n * W), o_ff = sz(sizeof(FieldFrame) * n);
    const size_t o_res = sz(sizeof(epid_field_result) * n);
    const size_t o_gh = sz(sizeof(double) * (size_t)(2 * lw_h + 1)), o_gv = sz(sizeof(double) * (size_t)(2 * lw_v + 1));
    // the 1-D stages run in chunks of frames so that the work areas (~1 MB per profile) stay bounded
    const int chunk = n < 256 ? n : 256;
    const size_t o_wk = sz(sizeof(double) * (size_t)chunk * 2 * hc.stride);
    int rc = ensure_scratch(ctx, o);
    if (rc != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    FieldConst* d_cst = (FieldConst*)(base + o_cst);
    FrameRef* d_rf = (FrameRef*)(base + o_rf);
    FrameStats* d_st = (FrameStats*)(base + o_st);
    uint32_t* d_rs = (uint32_t*)(base + o_rs);
    uint32_t* d_cs = (uint32_t*)(base + o_cs);
    FieldFrame* d_ff = (FieldFrame*)(base + o_ff);
    epid_field_result* d_res = (epid_field_result*)(base + o_res);
    double* d_gh = (double*)(base + o_gh);
    double* d_gv = (double*)(base + o_gv);
    double* d_wk = (double*)(base + o_wk);
    cudaStream_t st = ctx->stream;
    EPID_CUDA(cudaMemcpyAsync(d_cst, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    if (p->edge != 0) {
        EPID_CUDA(cudaMemcpyAsync(d_gh, gauss_h, sizeof(double) * (size_t)(2 * lw_h + 1), cudaMemcpyHostToDevice, st));
        EPID_CUDA(cudaMemcpyAsync(d_gv, gauss_v, sizeof(double) * (size_t)(2 * lw_v + 1), cudaMemcpyHostToDevice, st));
    }
    EPID_CUDA(cudaMemsetAsync(d_res, 0, sizeof(epid_field_result) * n, st));
    launch_refs_from_batch(ctx, st, (const uint16_t*)frames->dptr, n, H, W, 0, 0, d_rf);
    StatsGeom g;
    rc = make_stats_geom(&g, H, W);
    if (rc != EPID_OK) return rc;
    g.nranks = 6;
    g.ranks[0] = hc.p5.prev; g.ranks[1] = hc.p5.next;
    g.ranks[2] = hc.p50.prev; g.ranks[3] = hc.p50.next;
    g.ranks[4] = hc.p95.prev; g.ranks[5] = hc.p95.next;
    g.box = 0;
    rc = launch_frame_stats_inversion(ctx, st, g, d_rf, n, d_st, d_rs, d_cs);
    if (rc != EPID_OK) return rc;
    for (int c0 = 0; c0 < n; c0 += chunk) {
        const int cn = n - c0 < chunk ? n - c0 : chunk;
        dim3 grid(cn, 2);
        k_field_center<<<grid, FA_THREADS, 0, st>>>(d_cst, d_st + c0, d_rs + (size_t)c0 * H, d_cs + (size_t)c0 * W, d_ff + c0, d_wk, d_res + c0);
        k_field_strips<<<grid, FA_THREADS, 0, st>>>(d_cst, d_rf + c0, d_ff + c0, d_wk);
        k_field_profile<<<grid, FA_THREADS, 0, st>>>(d_cst, d_gh, d_gv, d_wk, d_res + c0);
        ctx->launches += 3;
    }
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaMemcpyAsync(results, d_res, sizeof(epid_field_result) * n, cudaMemcpyDeviceToHost, st));
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("field analysis pipeline failed: %s", cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    return EPID_OK;
}

extern "C" int32_t epid_single_profile(epid_ctx* ctx, const double* values, const double* x_values, int32_t n0, const epid_sp_params* p, const double* gauss,
                                       int32_t lw, int32_t n_expect, double fwxm_x, double pen_lower, double pen_upper,
                                       double in_field_ratio, double slope_exclusion_ratio, epid_sp_result* result, double* values_out,
                                       double* field_values_out, int32_t cap) {
    EPID_REQUIRE(ctx && values && p && result && values_out && field_values_out, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(n0 >= 3, EPID_ERR_INVALID, "profile too short");
    EPID_REQUIRE(p->edge != 1 || gauss, EPID_ERR_INVALID, "gaussian weights missing");
    EPID_REQUIRE(p->interpolation >= 0 && p->interpolation <= 2, EPID_ERR_INVALID, "interpolation code %d", p->interpolation);
    EPID_REQUIRE(p->interpolation != 2 || p->x_stop > p->x_start, EPID_ERR_INVALID, "pre-sampled profile needs x_stop > x_start");
    EPID_REQUIRE(!x_values || p->interpolation == 2, EPID_ERR_INVALID, "explicit abscissae need interpolation == 2");
    EPID_REQUIRE(fwxm_x >= 0 && fwxm_x <= 100, EPID_ERR_INVALID, "x must be between 0 and 100");
    EPID_REQUIRE(pen_lower <= pen_upper, EPID_ERR_INVALID, "Upper penumbra value must be larger than the lower penumbra value");
    EPID_CUDA(cudaSetDevice(ctx->device));
    int n = n0;
    if (p->interpolation == 1) n = (int)rint(p->dpmm > 0 ? (double)n0 / (p->dpmm * p->interpolation_resolution_mm) : (double)n0 * p->interpolation_factor);
    EPID_REQUIRE(n >= 3 && n <= cap, EPID_ERR_INVALID, "output capacity %d too small for %d samples", cap, n);
    const int nmax = n + 16;
    int pcap = 1;
    while (pcap < nmax / 2 + 8) pcap <<= 1;
    size_t o = 0;
    auto sz = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    const size_t o_x = sz(sizeof(double) * n0);
    const size_t o_raw = sz(sizeof(double) * n0), o_gw = sz(sizeof(double) * (size_t)(2 * lw + 1)), o_res = sz(sizeof(epid_sp_result));
    const size_t o_val = sz(sizeof(double) * n), o_fv = sz(sizeof(double) * n), o_wk = sz(sizeof(double) * (3 * (size_t)nmax + 8 * (size_t)pcap));
    int rc = ensure_scratch(ctx, o);
    if (rc != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    cudaStream_t st = ctx->stream;
    EPID_CUDA(cudaMemcpyAsync(base + o_raw, values, sizeof(double) * n0, cudaMemcpyHostToDevice, st));
    if (x_values) EPID_CUDA(cudaMemcpyAsync(base + o_x, x_values, sizeof(double) * n0, cudaMemcpyHostToDevice, st));
    if (p->edge == 1) EPID_CUDA(cudaMemcpyAsync(base + o_gw, gauss, sizeof(double) * (size_t)(2 * lw + 1), cudaMemcpyHostToDevice, st));
    k_single_profile<<<1, FA_THREADS, 0, st>>>(*p, (const double*)(base + o_raw), x_values ? (const double*)(base + o_x) : nullptr, n0, nmax, pcap, (const double*)(base + o_gw), lw, n_expect, fwxm_x,
                                               pen_lower, pen_upper, in_field_ratio, slope_exclusion_ratio, (double*)(base + o_wk),
                                               (epid_sp_result*)(base + o_res), (double*)(base + o_val), (double*)(base + o_fv));
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    EPID_CUDA(cudaMemcpyAsync(result, base + o_res, sizeof(epid_sp_result), cudaMemcpyDeviceToHost, st));
    EPID_CUDA(cudaStreamSynchronize(st));
    EPID_CUDA(cudaMemcpyAsync(values_out, base + o_val, sizeof(double) * result->n, cudaMemcpyDeviceToHost, st));
    if (result->fd_field_values_n > 0)
        EPID_CUDA(cudaMemcpyAsync(field_values_out, base + o_fv, sizeof(double) * result->fd_field_values_n, cudaMemcpyDeviceToHost, st));
    EPID_CUDA(cudaStreamSynchronize(st));
    return EPID_OK;
}
