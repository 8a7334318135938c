// Stencil kernels (internal interface).
#pragma once
#include "common.cuh"
#include "stats.cuh"

namespace epid {

// Per-frame value map applied while reading the source of a stencil:  v' = inv ? (mx + mn - v) : v
// (array_utils.invert, core/array_utils.py:75-77, materialised on the fly).
struct ValueMap {
    int inv;
    uint32_t mn, mx;
};

// scipy.ndimage.median_filter(size=k) semantics on uint16 views (mode='reflect', rank k*k/2, window offsets
// -(k/2) .. k-1-k/2).  For each i < n: src[i] (view H x W) -> dst[i] (compact, pitch dst_pitch).
// `select` (device, may be null): only frames with select[i] != 0 are processed.  maps (device, may be null).
int launch_median_u16(epid_ctx* ctx, cudaStream_t stream, const FrameRef* d_src, const FrameRef* d_dst, const ValueMap* d_maps,
                      const int* d_select, int n, int H, int W, int k);

// One scipy.ndimage.correlate1d pass over n compact float64 H x W frames on ctx->stream (filters.cu's k_correlate1d): weights w[2r + 1]
// on the host, mode 'reflect' (nearest == 0) or 'nearest' (nearest == 1).  Asynchronous; returns a launch error.
int correlate1d_f64(epid_ctx* ctx, const double* in, double* out, int n, int H, int W, int axis, const double* w, int r, int nearest);

}  // namespace epid
