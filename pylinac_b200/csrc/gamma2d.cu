// gamma_2d (reference core/gamma.py:229-330; Low et al. 2004, Table I) for a batch of (reference, evaluation) pairs.
//
//   dose_ta = dose_frac * reference.max()   (global)   or   dose_frac * reference   (local, elementwise)
//   eval_n = evaluation / dose_ta;  ref_n = reference / dose_ta
//   ref_n is nan or ref_n < threshold                         -> fill_value
//   G2 = nanmin over the disk of  dist_r_2[k] + d * d,  d = eval_n[clamp(y + dr[k]), clamp(x + dc[k])] - ref_n[y, x]
//   G2 >= cap**2 -> cap, else sqrt(G2)          (an all-nan disk gives nan: nan >= cap**2 is false and sqrt(nan) is nan)
//
// np.pad(eval_n, dta, mode="edge") is the row / column clamp to the evaluation's own shape, which may be larger than the reference's.
// Types follow numpy 2: TR is the type of dose_ta and ref_n (float32 for a float32 reference, whose max() is an np.float32 and whose
// python-float factors are weak; float64 otherwise), TE = result_type(evaluation, TR) is the type of eval_n, of d and of d * d; the sum
// with the fp64 distance is fp64.  -fmad=false, IEEE division in the reference's order and __dsqrt_rn make every map bit-identical.
//
// Three launches: the per-pair max (global mode), the normalisation into scratch, and the search.  The host sorts the disk offsets by
// dist_r_2 (raster order breaks ties), so a thread can stop at offset k once it has seen a non-nan term and dist_r_2[k] >=
// min(best, cap**2): every later term is >= dist_r_2[k] because fl(a + b) >= a for b >= 0, so neither the minimum nor the capped
// output can change.  full_search != 0 visits the whole disk (the A/B check of that argument).
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace epid {
namespace {

__device__ __forceinline__ double g2_load(const void* p, int dt, size_t i) {   // exact for every dtype but int64 (rounded as numpy)
    switch (dt) {
        case EPID_U8: return ((const uint8_t*)p)[i];
        case EPID_U16: return ((const uint16_t*)p)[i];
        case EPID_I16: return ((const int16_t*)p)[i];
        case EPID_I32: return ((const int32_t*)p)[i];
        case EPID_I64: return (double)((const long long*)p)[i];
        case EPID_F32: return ((const float*)p)[i];
        default: return ((const double*)p)[i];
    }
}

// ndarray.max() of each reference frame: a nan anywhere gives nan
__global__ void __launch_bounds__(1024) k_gamma2d_max(const void* __restrict__ ref, int dt, size_t per, double* __restrict__ mx) {
    const size_t base = (size_t)blockIdx.x * per;
    double m = -INFINITY;
    for (size_t i = threadIdx.x; i < per; i += blockDim.x) {
        const double v = g2_load(ref, dt, base + i);
        if (isnan(v) || v > m) m = isnan(m) ? m : v;
    }
    __shared__ double part[32];
    for (int o = 16; o > 0; o >>= 1) {
        const double v = __shfl_xor_sync(0xffffffffu, m, o);
        if (isnan(v) || v > m) m = isnan(m) ? m : v;
    }
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < (int)(blockDim.x >> 5); k++) {
            const double v = part[k];
            if (isnan(v) || v > m) m = isnan(m) ? m : v;
        }
        mx[blockIdx.x] = m;
    }
}

// eval_n over the evaluation's n x he x we elements, ref_n over the reference's n x h x w (local mode: equal shapes)
template <class TR, class TE>
__global__ void k_gamma2d_norm(const void* __restrict__ ref, int rdt, const void* __restrict__ ev, int edt, size_t rper, size_t eper,
                               int n, double dose_frac, const double* __restrict__ mx, int global_dose, TR* __restrict__ ref_n,
                               TE* __restrict__ eval_n) {
    const size_t total = (size_t)n * eper;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t f = i / eper;
        const TR dta = (TR)dose_frac * (global_dose ? (TR)mx[f] : (TR)g2_load(ref, rdt, i));
        eval_n[i] = (TE)g2_load(ev, edt, i) / (TE)dta;
        if (i - f * eper < rper) {
            const size_t j = f * rper + (i - f * eper);
            const TR dr = global_dose ? dta : (TR)dose_frac * (TR)g2_load(ref, rdt, j);
            ref_n[j] = (TR)g2_load(ref, rdt, j) / dr;
        }
    }
}

// thread per reference pixel; offs: int4 {dr, dc, lo, hi word of dist_r_2}, sorted by dist_r_2
template <class TR, class TE>
__global__ void __launch_bounds__(256) k_gamma2d(const TR* __restrict__ ref_n, const TE* __restrict__ eval_n, const int4* __restrict__ offs,
                                                 int n_off, int h, int w, int he, int we, TR thr, double cap, double cap2, double fill,
                                                 int full_search, double* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
    if (x >= w || y >= h) return;
    const size_t o = ((size_t)f * h + y) * w + x;
    const TR r = ref_n[o];
    if (isnan(r) || r < thr) {
        out[o] = fill;
        return;
    }
    const TE* e = eval_n + (size_t)f * he * we;
    double best = 0.0;
    bool seen = false;
    for (int k = 0; k < n_off; k++) {
        const int4 t = __ldg(offs + k);
        const double d2 = __hiloint2double(t.w, t.z);
        if (!full_search && seen && d2 >= fmin(best, cap2)) break;
        const int er = min(max(y + t.x, 0), he - 1), ec = min(max(x + t.y, 0), we - 1);
        const TE d = __ldg(e + (size_t)er * we + ec) - (TE)r;
        const double v = d2 + (double)(d * d);
        if (!isnan(v) && (!seen || v < best)) {
            best = v;
            seen = true;
        }
    }
    out[o] = !seen ? (double)NAN : (best >= cap2 ? cap : __dsqrt_rn(best));
}

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

template <class TR, class TE>
int run(epid_ctx* ctx, const epid_batch* ref, const epid_batch* ev, double dose_frac, double threshold, double cap, double cap2,
        double fill_value, int global_dose, const std::vector<int4>& table, int full_search, epid_batch* out) {
    const int n = ref->n, h = ref->h, w = ref->w, he = ev->h, we = ev->w;
    const size_t rper = (size_t)h * w, eper = (size_t)he * we;
    const size_t sz_t = al256(sizeof(int4) * table.size()), sz_m = al256(8 * (size_t)n), sz_r = al256(sizeof(TR) * n * rper);
    int rc = ensure_scratch(ctx, sz_t + sz_m + sz_r + sizeof(TE) * n * eper);
    if (rc != EPID_OK) return rc;
    char* p = (char*)ctx->scratch;
    int4* d_tab = (int4*)p; p += sz_t;
    double* d_max = (double*)p; p += sz_m;
    TR* d_ref = (TR*)p; p += sz_r;
    TE* d_ev = (TE*)p;
    cudaStream_t s = ctx->stream;
    EPID_CUDA(cudaMemcpyAsync(d_tab, table.data(), sizeof(int4) * table.size(), cudaMemcpyHostToDevice, s));
    if (global_dose) {
        k_gamma2d_max<<<n, 1024, 0, s>>>(ref->dptr, ref->dtype, rper, d_max);
        ctx->launches++;
    }
    const size_t total = (size_t)n * eper;
    const int grid = (int)std::min<size_t>((total + 255) / 256, (size_t)ctx->sm_count * 16);
    k_gamma2d_norm<TR, TE><<<grid, 256, 0, s>>>(ref->dptr, ref->dtype, ev->dptr, ev->dtype, rper, eper, n, dose_frac, d_max, global_dose,
                                                d_ref, d_ev);
    const dim3 block(32, 8), tiles((w + 31) / 32, (h + 7) / 8, n);
    k_gamma2d<TR, TE><<<tiles, block, 0, s>>>(d_ref, d_ev, d_tab, (int)table.size(), h, w, he, we, (TR)threshold, cap, cap2, fill_value,
                                              full_search, (double*)out->dptr);
    ctx->launches += 2;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("gamma_2d kernels failed: %s", cudaGetErrorString(e)); return EPID_ERR_CUDA; }
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_gamma2d(epid_ctx* ctx, const epid_batch* ref, const epid_batch* eval, double dose_frac, double threshold, double cap,
                                double cap2, double fill_value, int32_t global_dose, const int32_t* offsets, const double* dist2, int32_t n_off,
                                int32_t full_search, epid_batch** out) {
    EPID_REQUIRE(ctx && ref && eval && offsets && dist2 && out, EPID_ERR_INVALID, "NULL argument");
    EPID_REQUIRE(n_off > 0, EPID_ERR_INVALID, "empty offset table");
    EPID_REQUIRE(dtype_size(ref->dtype) > 0 && dtype_size(eval->dtype) > 0, EPID_ERR_INVALID, "unknown dtype");
    EPID_REQUIRE(ref->n == eval->n, EPID_ERR_INVALID, "%d reference frames but %d evaluation frames", ref->n, eval->n);
    if (global_dose)
        EPID_REQUIRE(eval->h >= ref->h && eval->w >= ref->w, EPID_ERR_INVALID,
                     "the evaluation (%d x %d) is smaller than the reference (%d x %d)", eval->h, eval->w, ref->h, ref->w);
    else
        EPID_REQUIRE(eval->h == ref->h && eval->w == ref->w, EPID_ERR_INVALID,
                     "local dose needs equal shapes: reference %d x %d, evaluation %d x %d", ref->h, ref->w, eval->h, eval->w);
    EPID_CUDA(cudaSetDevice(ctx->device));
    std::vector<int4> table(n_off);
    for (int k = 0; k < n_off; k++) {
        uint32_t words[2];
        std::memcpy(words, dist2 + k, 8);
        table[k] = make_int4(offsets[2 * k], offsets[2 * k + 1], (int)words[0], (int)words[1]);
    }
    int rc = epid_batch_alloc(ctx, EPID_F64, ref->n, ref->h, ref->w, out);
    if (rc != EPID_OK) return rc;
    // numpy 2: a float32 reference keeps dose_ta / ref_n in float32; eval_n is float32 only if the evaluation's dtype fits float32
    const bool r32 = ref->dtype == EPID_F32;
    const bool e32 = r32 && (eval->dtype == EPID_F32 || eval->dtype == EPID_U8 || eval->dtype == EPID_U16 || eval->dtype == EPID_I16);
    if (e32)
        rc = run<float, float>(ctx, ref, eval, dose_frac, threshold, cap, cap2, fill_value, global_dose, table, full_search, *out);
    else if (r32)
        rc = run<float, double>(ctx, ref, eval, dose_frac, threshold, cap, cap2, fill_value, global_dose, table, full_search, *out);
    else
        rc = run<double, double>(ctx, ref, eval, dose_frac, threshold, cap, cap2, fill_value, global_dose, table, full_search, *out);
    if (rc != EPID_OK) {
        epid_batch_free(*out);
        *out = nullptr;
    }
    return rc;
}
