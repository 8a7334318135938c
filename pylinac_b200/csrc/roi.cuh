// Pixel-selection rules shared by the ROI kernels (roi.cu, vmat.cu) and the CT localization (ct.cu): skimage.draw.disk's bounding box,
// and the point-in-quadrilateral rule of RectangleROI.pixels_flat (core/roi.py:641-660 -> skimage.draw.polygon): integer pixel
// coordinates inside the corner polygon or ON its boundary.
#pragma once

#include <cmath>

namespace epid {

// skimage.draw.disk's bounding box of one disk: rows r0 .. r0 + bh - 1, columns c0 .. c0 + bw - 1 (bh, bw >= 0)
struct DiskBox { long long r0, c0, bh, bw; };
__host__ __device__ inline DiskBox disk_box(double cy, double cx, double R) {
    R = fabs(R);                                     // skimage's rotated radius |r cos 0| + r sin 0
    DiskBox b;
    b.r0 = (long long)ceil(cy - R);
    b.c0 = (long long)ceil(cx - R);
    b.bh = (long long)floor(cy + R) - b.r0 + 1;
    b.bw = (long long)floor(cx + R) - b.c0 + 1;
    if (b.bh < 0) b.bh = 0;
    if (b.bw < 0) b.bw = 0;
    return b;
}

// 0 outside, non-zero inside or on the boundary (crossing number with explicit edge / vertex tests, the structure of skimage's
// _geometry.point_in_polygon)
__device__ inline int point_in_quad(const double* vx, const double* vy, double x, double y) {
    int r = 0;
    double x0 = vx[3] - x, y0 = vy[3] - y;
    for (int i = 0; i < 4; i++) {
        const double x1 = vx[i] - x, y1 = vy[i] - y;
        if (y1 == 0 && (x1 == 0 || (y0 == 0 && ((x1 > 0) == (x0 < 0))))) return 2;      // vertex, or on a horizontal edge
        if ((y1 < 0) != (y0 < 0)) {      // the edge crosses the horizontal line through the point
            if (x0 >= 0) {
                if (x1 > 0) r += 1;                       // entirely to the right
                else {
                    const double det = (x0 * y1 - x1 * y0);
                    if (det == 0) return 3;               // on the edge
                    if ((det > 0) == (y1 > y0)) r += 1;
                }
            } else if (x1 > 0) {
                const double det = (x0 * y1 - x1 * y0);
                if (det == 0) return 3;
                if ((det > 0) == (y1 > y0)) r += 1;
            }
        }
        x0 = x1;
        y0 = y1;
    }
    return r & 1;
}

}  // namespace epid
