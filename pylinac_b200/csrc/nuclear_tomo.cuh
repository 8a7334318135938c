// The sphere search of pylinac.nuclear.TomographicContrast (nuclear.py:1714-1724): scipy 1.18.1's _minimize_neldermead in 3-D with
// minimize()'s defaults and bounds, and the 4-key argsort it sorts the simplex with.  Shared by the device kernel of nuclear_tomo.cu
// and the host check tests/nt_nm_check.cu, so that the host build settles the search against scipy before any device run.
//
// Build with FMA contraction off (-fmad=false on the device, -ffp-contract=off on the host): every expression rounds as numpy's.
#pragma once
#include <cmath>

#ifdef __CUDACC__
#define NT_HD __host__ __device__ __forceinline__
#else
#define NT_HD inline
#endif

namespace epid {
namespace nt {

// np.argsort (default kind) of 4 float64 keys as numpy 2.3 runs it on an AVX-512 (AVX512_SKX) host, where it dispatches to the
// x86-simd-sort network, which is not stable.  Keys with a nan sort stably, nans last.  Without a nan the network gives a stable
// sort except on 5 weak orderings, found by comparing np.argsort with a stable sort on every weak ordering of 4 keys (DESIGN.md
// section 4.15).  A weak ordering is written as each key's count of strictly smaller keys, in base 5, key 0 first.
NT_HD void argsort4(const double f[4], int ind[4]) {
    bool nan = false;
    for (int i = 0; i < 4; i++) nan |= f[i] != f[i];
    if (!nan) {
        int code = 0;
        for (int i = 0; i < 4; i++) {
            int below = 0;
            for (int j = 0; j < 4; j++) below += f[j] < f[i];
            code = code * 5 + below;
        }
        //                           (2,2,0,0)     (2,3,0,0)     (3,2,0,0)     (2,2,0,1)     (2,2,1,0)
        const int codes[5] = {300, 325, 425, 301, 305};
        const int perms[5][4] = {{3, 2, 1, 0}, {3, 2, 0, 1}, {3, 2, 1, 0}, {2, 3, 1, 0}, {3, 2, 1, 0}};
        for (int k = 0; k < 5; k++) {
            if (code == codes[k]) {
                for (int i = 0; i < 4; i++) ind[i] = perms[k][i];
                return;
            }
        }
    }
    // stable insertion sort, nans last
    for (int i = 0; i < 4; i++) ind[i] = i;
    for (int i = 1; i < 4; i++) {
        const int v = ind[i];
        int j = i - 1;
        for (; j >= 0; j--) {
            const double a = f[v], b = f[ind[j]];
            const bool less = (b != b) ? (a == a) : (a < b);
            if (!less) break;
            ind[j + 1] = ind[j];
        }
        ind[j + 1] = v;
    }
}

// create_sphere_mask (nuclear.py:1825-1835) at voxel (x, y, z): ((x - col)**2 + (y - row)**2) + (z - zed)**2 <= radius**2, with
// r2 = radius**2 as Python computes it
NT_HD bool in_sphere(int x, int y, int z, double col, double row, double zed, double r2) {
    const double dx = (double)x - col, dy = (double)y - row, dz = (double)z - zed;
    return (dx * dx + dy * dy) + dz * dz <= r2;
}

// [lo, hi] along one axis of length n: every index the sphere can reach, clipped to the volume (lo > hi: none)
NT_HD void sphere_span(double c, double r2, int n, int& lo, int& hi) {
    const double r = sqrt(r2) + 1;
    const double a = floor(c - r), b = ceil(c + r);
    lo = a < 0 ? 0 : (a > n ? n : (int)a);
    hi = b > n - 1 ? n - 1 : (b < -1 ? -1 : (int)b);
}

// contrast_f (nuclear.py:1850-1856) from the sphere's exact sum and count: -michelson([nanmean, baseline]) * 100.  An empty sphere's
// mean is nan, which michelson ignores.
NT_HD double contrast(unsigned long long sum, long long count, double baseline) {
    const double mean = count ? (double)sum / (double)count : NAN;
    double mx, mn;
    if (mean != mean) {
        mx = mn = baseline;
    } else if (baseline != baseline) {
        mx = mn = mean;
    } else {
        mx = mean > baseline ? mean : baseline;
        mn = mean < baseline ? mean : baseline;
    }
    return -((mx - mn) / (mx + mn)) * 100;
}

// np.clip(x, lo, hi) = minimum(maximum(x, lo), hi), nan propagating
NT_HD double clip(double x, double lo, double hi) {
    if (x != x) return x;
    const double t = x < lo ? lo : x;
    return t > hi ? hi : t;
}

struct Search {
    double x[3];        // res.x
    double fun;         // res.fun = np.min(fsim)
    int nfev, nit;
    int status;         // 0 converged, 1 maxfev, 2 maxiter (scipy's warnflag)
};

struct Simplex {
    double sim[4][3];
    double fsim[4];
};

NT_HD void sort_simplex(Simplex& s) {
    int ind[4];
    argsort4(s.fsim, ind);
    Simplex t = s;
    for (int i = 0; i < 4; i++) {
        s.fsim[i] = t.fsim[ind[i]];
        for (int k = 0; k < 3; k++) s.sim[i][k] = t.sim[ind[i]][k];
    }
}

// _minimize_neldermead(func, x0, bounds=(lb, ub), maxiter, maxfev) with xatol = fatol = 1e-4, rho, chi, psi, sigma = 1, 2, 1/2, 1/2.
// func(const double x[3]) -> double is called with every thread of a CTA at once on the device (it reduces across the CTA); the
// bookkeeping here is uniform, so every thread takes the same path.  func is not called once maxfun calls were made: that is
// scipy's _MaxFuncCallError, which abandons the rest of the current step.
template <class F>
NT_HD Search nelder_mead(const double x0in[3], const double lb[3], const double ub[3], int maxfun, int maxiter, F& func) {
    const double xatol = 1e-4, fatol = 1e-4;
    Simplex s;
    double x0[3];
    for (int k = 0; k < 3; k++) x0[k] = clip(x0in[k], lb[k], ub[k]);
    for (int j = 0; j < 4; j++)
        for (int k = 0; k < 3; k++) s.sim[j][k] = x0[k];
    for (int k = 0; k < 3; k++) s.sim[k + 1][k] = x0[k] != 0 ? (1 + 0.05) * x0[k] : 0.00025;
    for (int j = 0; j < 4; j++) {
        for (int k = 0; k < 3; k++) {
            double v = s.sim[j][k];
            if (v > ub[k]) v = 2 * ub[k] - v;      // reflect into the interior, then clip
            s.sim[j][k] = clip(v, lb[k], ub[k]);
        }
        s.fsim[j] = INFINITY;
    }
    int fcalls = 0;
    auto call = [&](const double* x, double* out) -> bool {
        if (fcalls >= maxfun) return false;
        fcalls++;
        *out = func(x);
        return true;
    };
    for (int j = 0; j < 4; j++)
        if (!call(s.sim[j], &s.fsim[j])) break;
    sort_simplex(s);
    sort_simplex(s);

    int iterations = 1;
    while (fcalls < maxfun && iterations < maxiter) {
        double dx = 0, df = 0;                     // np.max propagates a nan
        for (int j = 1; j < 4; j++) {
            for (int k = 0; k < 3; k++) {
                const double d = fabs(s.sim[j][k] - s.sim[0][k]);
                dx = (d != d || dx != dx) ? NAN : (d > dx ? d : dx);
            }
            const double d = fabs(s.fsim[0] - s.fsim[j]);
            df = (d != d || df != df) ? NAN : (d > df ? d : df);
        }
        if (dx <= xatol && df <= fatol) break;
        double xbar[3], xr[3];
        for (int k = 0; k < 3; k++) {
            xbar[k] = ((s.sim[0][k] + s.sim[1][k]) + s.sim[2][k]) / 3;
            xr[k] = clip(2 * xbar[k] - s.sim[3][k], lb[k], ub[k]);
        }
        double fxr;
        bool ok = call(xr, &fxr);
        if (ok) {
            if (fxr < s.fsim[0]) {
                double xe[3], fxe;
                for (int k = 0; k < 3; k++) xe[k] = clip(3 * xbar[k] - 2 * s.sim[3][k], lb[k], ub[k]);
                ok = call(xe, &fxe);
                if (ok) {
                    const bool e = fxe < fxr;
                    for (int k = 0; k < 3; k++) s.sim[3][k] = e ? xe[k] : xr[k];
                    s.fsim[3] = e ? fxe : fxr;
                }
            } else if (fxr < s.fsim[2]) {
                for (int k = 0; k < 3; k++) s.sim[3][k] = xr[k];
                s.fsim[3] = fxr;
            } else {
                bool shrink;
                double xc[3], fxc;
                if (fxr < s.fsim[3]) {
                    for (int k = 0; k < 3; k++) xc[k] = clip(1.5 * xbar[k] - 0.5 * s.sim[3][k], lb[k], ub[k]);
                    ok = call(xc, &fxc);
                    shrink = !(fxc <= fxr);
                } else {
                    for (int k = 0; k < 3; k++) xc[k] = clip(0.5 * xbar[k] + 0.5 * s.sim[3][k], lb[k], ub[k]);
                    ok = call(xc, &fxc);
                    shrink = !(fxc < s.fsim[3]);
                }
                if (ok && !shrink) {
                    for (int k = 0; k < 3; k++) s.sim[3][k] = xc[k];
                    s.fsim[3] = fxc;
                }
                if (ok && shrink) {
                    for (int j = 1; j < 4 && ok; j++) {
                        for (int k = 0; k < 3; k++)
                            s.sim[j][k] = clip(s.sim[0][k] + 0.5 * (s.sim[j][k] - s.sim[0][k]), lb[k], ub[k]);
                        ok = call(s.sim[j], &s.fsim[j]);
                    }
                }
            }
        }
        if (ok) iterations++;
        sort_simplex(s);
    }
    Search r;
    for (int k = 0; k < 3; k++) r.x[k] = s.sim[0][k];
    double fmin = s.fsim[0];                       // np.min propagates a nan
    for (int j = 1; j < 4; j++) fmin = (fmin != fmin || s.fsim[j] != s.fsim[j]) ? NAN : (s.fsim[j] < fmin ? s.fsim[j] : fmin);
    r.fun = fmin;
    r.nfev = fcalls;
    r.nit = iterations;
    r.status = fcalls >= maxfun ? 1 : (iterations >= maxiter ? 2 : 0);
    return r;
}

}  // namespace nt
}  // namespace epid
