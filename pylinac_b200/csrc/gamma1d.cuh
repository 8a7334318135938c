// The per-point arithmetic of gamma_geometric (reference core/gamma.py:16-226), shared by the device kernels of gamma1d.cu and the host
// check tests/gamma1d_dist_check.cu, so that the host build settles its rounding against Python before any device run.
#pragma once
#include <cfloat>
#include <cmath>

#ifdef __CUDACC__
#define G1_HD __host__ __device__ __forceinline__
#else
#define G1_HD inline
#endif

namespace epid {
namespace g1 {

// CPython 3.12 math.dist of two 2-D points (Modules/mathmodule.c, vector_norm): the squares of the scaled differences summed in
// double-double, a square root, and one differential correction from the residual.  Python's min() order of special cases: an
// infinite difference wins over a nan, and a zero maximum returns zero.

// csum += x * y in double-double: the square is exact, the sum exact as |csum| >= |hi|, and the two low parts accumulate
G1_HD void dl_add_square(double x, double y, double& csum, double& frac1, double& frac2) {
    const double hi = x * y, lo = fma(x, y, -hi);
    const double s = csum + hi;
    frac2 += (csum - s) + hi;
    frac1 += lo;
    csum = s;
}

G1_HD double py_norm2(double a, double b, double mx) {
    int e = ilogb(mx) + 1;               // frexp's exponent
    double unscale = 1.0;
    if (e < -1023) {                     // subnormal maximum: ldexp(1, -e) would overflow; CPython rescales by DBL_MIN first
        a /= DBL_MIN;
        b /= DBL_MIN;
        mx /= DBL_MIN;
        unscale = DBL_MIN;
        e = ilogb(mx) + 1;
    }
    const double scale = ldexp(1.0, -e);
    double csum = 1.0, frac1 = 0.0, frac2 = 0.0;
    dl_add_square(a * scale, a * scale, csum, frac1, frac2);
    dl_add_square(b * scale, b * scale, csum, frac1, frac2);
    double h = sqrt(csum - 1.0 + (frac1 + frac2));
    dl_add_square(-h, h, csum, frac1, frac2);
    const double x = csum - 1.0 + (frac1 + frac2);
    h += x / (2.0 * h);
    return unscale * (h / scale);
}

G1_HD double py_dist(double px, double py, double qx, double qy) {
    const double a = fabs(px - qx), b = fabs(py - qy);
    double mx = 0.0;
    if (a > mx) mx = a;
    if (b > mx) mx = b;
    if (isinf(mx)) return mx;
    if (isnan(a) || isnan(b)) return NAN;
    if (mx == 0.0) return mx;
    return py_norm2(a, b, mx);
}

// _compute_distance(p, [v1, v2]): V = v1 - v2, P = p - v2; V^T V and V^T P are the 2-element BLAS dot products, which round as
// fma(x1, y1, x0 * y0); pinv of the 1 x 1 V^T V is 1 / vtv (0 for 0).  A negative weight gives Python's min of the two vertex
// distances, otherwise the norm of p minus the projection (the projection itself unfused).  *svd_fail is set where vtv is nan,
// for which numpy's pinv raises LinAlgError("SVD did not converge").
G1_HD double segment_distance(double px, double py, double v1x, double v1y, double v2x, double v2y, bool* svd_fail) {
    const double a0 = v1x - v2x, a1 = v1y - v2y, p0 = px - v2x, p1 = py - v2y;
    const double vtv = fma(a1, a1, a0 * a0);
    if (isnan(vtv)) {
        *svd_fail = true;
        return NAN;
    }
    const double inv = vtv == 0.0 ? 0.0 : 1.0 / vtv;
    const double w0 = inv * fma(a1, p1, a0 * p0);
    const double w1 = 1.0 - w0;
    if (w0 < 0.0 || w1 < 0.0) {
        const double d1 = py_dist(px, py, v1x, v1y), d2 = py_dist(px, py, v2x, v2y);
        return d2 < d1 ? d2 : d1;
    }
    const double q0 = w0 * v1x + w1 * v2x, q1 = w0 * v1y + w1 * v2y;
    const double d0 = px - q0, d1 = py - q1;
    return sqrt(fma(d1, d1, d0 * d0));
}

// np.argmin(np.abs(x - t)) over a strictly monotonic x (increasing, or decreasing with dec): |fl(x[i] - t)| falls up to the first
// index p on t's far side and rises from there, so the minimum is at p - 1 or p, and the first index holding it (argmin's tie rule)
// is found by a second bisection over [0, p).
G1_HD int argmin_abs(const double* x, int m, double t, bool dec) {
    if (isnan(t)) return 0;
    int lo = 0, hi = m;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (dec ? x[mid] <= t : x[mid] >= t) hi = mid; else lo = mid + 1;
    }
    const int p = lo;
    double best = INFINITY;
    if (p < m) best = fabs(x[p] - t);
    if (p > 0 && fabs(x[p - 1] - t) < best) best = fabs(x[p - 1] - t);
    lo = 0;
    hi = p;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (fabs(x[mid] - t) <= best) hi = mid; else lo = mid + 1;
    }
    return lo;
}

}  // namespace g1
}  // namespace epid
