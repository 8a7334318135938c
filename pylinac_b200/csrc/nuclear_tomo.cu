// pylinac.nuclear.TomographicContrast (nuclear.py:1553-1856) on the device: the SPECT slice analysis and the bounded Nelder-Mead
// sphere search, bit-identical to the reference.
//
//   k_nt_max      one CTA per volume: the volume's maximum.
//   k_nt_slices   one CTA per slice, the slice in shared memory when 12 bytes per pixel fit (the global workspace otherwise; same
//                 code): the threshold at 10 % of the volume's maximum (compared in float64, as numpy promotes it), then the stages of
//                 nuclear_stages.cuh shared with k_nm_frame and k_tu_frame: 4-connected labelling, the largest region's area, bounding
//                 box and exact coordinate sums, and one exact squared EDT of the whole binary; the FOV against erosion / 2, and the
//                 Michelson ratio, exact sum and count of the eroded pixels.
//   k_nt_spheres  one CTA per (volume, sphere): scipy's _minimize_neldermead (nuclear_tomo.cuh), each objective evaluation an exact
//                 sum and count over the sphere's bounding box, then the sum, count and min at res.x.
//
// Exactness (DESIGN.md section 4.15): the volumes are integer counts, so every sum is an exact integer below 2^53, every mean and
// ratio rounds once, and the search's arithmetic is scipy's expression order without FMA (-fmad=false).
#include "common.cuh"
#include "nuclear_stages.cuh"
#include "nuclear_tomo.cuh"

#include <cmath>

namespace epid {
namespace {

using namespace nm;

constexpr int NT_THREADS = 512;
constexpr int NT_SPHERE_THREADS = 128;

__global__ void __launch_bounds__(NT_THREADS) k_nt_max(const uint16_t* __restrict__ vol, size_t voxels, uint32_t* __restrict__ gmax) {
    __shared__ unsigned long long red[32];
    const uint16_t* v = vol + (size_t)blockIdx.x * voxels;
    unsigned long long m = 0;
    for (size_t i = threadIdx.x; i < voxels; i += blockDim.x) m = max(m, (unsigned long long)v[i]);
    m = block_reduce(m, OpMax(), red);
    if (threadIdx.x == 0) gmax[blockIdx.x] = (uint32_t)m;
}

__global__ void __launch_bounds__(NT_THREADS) k_nt_slices(const uint16_t* __restrict__ vol, int nz, int h, int w,
                                                          const uint32_t* __restrict__ gmax, double ufov_erode, uint32_t* ws,
                                                          epid_nt_slice* res) {
    extern __shared__ __align__(16) uint32_t dsm[];
    __shared__ unsigned long long red[32];
    const int f = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int N = h * w;
    const size_t fo = (size_t)f * N;
    uint32_t* S = ws ? ws + 3 * fo : dsm;
    int* P = (int*)(S + N);       // -1 / union-find parent; later the squared EDT
    int* A = (int*)(S + 2 * N);   // component areas; later the column distances of the EDT
    const uint16_t* src = vol + fo;
    epid_nt_slice r = {};

    // ---- arr[arr < volume.max() * 0.10] = 0; binary = arr > 0
    const double thr = (double)gmax[f / nz] * 0.10;
    for (int p = tid; p < N; p += nt) {
        const uint32_t v = src[p];
        S[p] = (double)v < thr ? 0u : v;
        P[p] = S[p] ? p : -1;
    }
    __syncthreads();

    label_areas(P, A, h, w);
    const Component c = largest_component(P, A, h, w, red);
    if (c.area == 0) {            // no label: slice_data skips the slice
        if (tid == 0) {
            r.status = EPID_NT_NO_COMPONENT;
            res[f] = r;
        }
        return;
    }
    const int erosion = (int)rint(ufov_erode * (double)c.longest);  // int(round(...)): Python rounds halves to even, as rint does
    r.longest = c.longest;
    r.erosion = erosion;
    r.centroid_row = (double)c.rsum / (double)c.area;               // skimage: the mean of the global coordinates
    r.centroid_col = (double)c.csum / (double)c.area;
    squared_edt(P, A, h, w, nullptr);

    // ---- the FOV: distance > erosion / 2  <=>  4 d^2 > erosion^2 (every pixel when the erosion is negative)
    const long long e2 = (long long)erosion * erosion;
    unsigned long long mx = 0, mn = ~0ull, sum = 0, cnt = 0;
    for (int p = tid; p < N; p += nt) {
        if (!(erosion < 0 || 4LL * P[p] > e2)) continue;
        mx = max(mx, (unsigned long long)S[p]);
        mn = min(mn, (unsigned long long)S[p]);
        sum += S[p];
        cnt++;
    }
    mx = block_reduce(mx, OpMax(), red);
    mn = block_reduce(mn, OpMin(), red);
    sum = block_reduce(sum, OpSum(), red);
    cnt = block_reduce(cnt, OpSum(), red);
    r.area = (int)cnt;
    r.sum = sum;
    if (cnt) {
        r.max = (int)mx;
        r.min = (int)mn;
        r.uniformity = (double)(mx - mn) / (double)(mx + mn);      // michelson of the FOV: exact integers, one rounding
        r.value = (double)sum / (double)cnt;                       // nanmean: an exact sum over the count, one rounding
    } else {
        r.uniformity = NAN;                                        // all-nan FOV: nanmax / nanmin / nanmean give nan
        r.value = NAN;
    }
    if (tid == 0) res[f] = r;
}

// sum, count and min of the voxels of the sphere (col, row, zed, r2) in one volume; every thread gets the result
__device__ void sphere_sum(const uint16_t* __restrict__ v, int nz, int h, int w, const double* x, double r2, unsigned long long* red,
                           unsigned long long* sum, unsigned long long* cnt, unsigned long long* mn) {
    int z0, z1, y0, y1, x0, x1;
    nt::sphere_span(x[2], r2, nz, z0, z1);
    nt::sphere_span(x[1], r2, h, y0, y1);
    nt::sphere_span(x[0], r2, w, x0, x1);
    const int bx = x1 - x0 + 1, by = y1 - y0 + 1, bz = z1 - z0 + 1;
    const long long nbox = bx > 0 && by > 0 && bz > 0 ? (long long)bx * by * bz : 0;
    unsigned long long s = 0, c = 0, m = ~0ull;
    for (long long q = threadIdx.x; q < nbox; q += blockDim.x) {
        const int xx = x0 + (int)(q % bx);
        const long long t = q / bx;
        const int yy = y0 + (int)(t % by), zz = z0 + (int)(t / by);
        if (!nt::in_sphere(xx, yy, zz, x[0], x[1], x[2], r2)) continue;
        const unsigned long long val = v[((size_t)zz * h + yy) * w + xx];
        s += val;
        c++;
        m = min(m, val);
    }
    *sum = block_reduce(s, OpSum(), red);
    *cnt = block_reduce(c, OpSum(), red);
    if (mn) *mn = block_reduce(m, OpMin(), red);
}

__global__ void __launch_bounds__(NT_SPHERE_THREADS) k_nt_spheres(const uint16_t* __restrict__ vol, int nz, int h, int w,
                                                                  const epid_nt_sphere_in* __restrict__ in, int maxfun, int maxiter,
                                                                  epid_nt_sphere* __restrict__ res) {
    __shared__ unsigned long long red[32];
    const epid_nt_sphere_in q = in[blockIdx.x];
    const uint16_t* v = vol + (size_t)q.volume * nz * h * w;
    int n_empty = 0;
    auto func = [&](const double* x) -> double {
        unsigned long long s, c;
        sphere_sum(v, nz, h, w, x, q.r2, red, &s, &c, nullptr);
        n_empty += c == 0;
        return nt::contrast(s, (long long)c, q.baseline);
    };
    const nt::Search s = nt::nelder_mead(q.x0, q.lb, q.ub, maxfun, maxiter, func);
    unsigned long long sum, cnt, mn;
    sphere_sum(v, nz, h, w, s.x, q.r2, red, &sum, &cnt, &mn);
    if (threadIdx.x == 0) {
        epid_nt_sphere r = {};
        for (int k = 0; k < 3; k++) r.x[k] = s.x[k];
        r.fun = s.fun;
        r.nfev = s.nfev;
        r.nit = s.nit;
        r.status = s.status;
        r.n_empty = n_empty;
        r.count = (int)cnt;
        r.min = cnt ? (int)mn : 0;
        r.sum = sum;
        res[blockIdx.x] = r;
    }
}

int nt_check(const epid_batch* volumes, int nz) {
    int rc = check_volumes(volumes, nz, "tomographic volumes");
    if (rc != EPID_OK) return rc;
    EPID_REQUIRE((long long)volumes->h * volumes->w < (1LL << 28), EPID_ERR_UNSUPPORTED, "slice %d x %d is too large", volumes->h,
                 volumes->w);
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_nt_slices(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, double ufov_erode, struct epid_nt_slice* results) {
    EPID_REQUIRE(ctx && results, EPID_ERR_INVALID, "NULL argument");
    int rc = nt_check(volumes, nz);
    if (rc != EPID_OK) return rc;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const int n = volumes->n, h = volumes->h, w = volumes->w, nvol = n / nz;
    if (n == 0) return EPID_OK;
    const size_t N = (size_t)h * w;
    // ctx->scratch: [volume maxima] [result rows] [per-slice workspace when the slice does not fit shared memory]
    FrameScratch s;
    if ((rc = frame_scratch(ctx, n, N, 12, 1024, nvol * sizeof(uint32_t), n * sizeof(epid_nt_slice), 0, &s)) != EPID_OK) return rc;
    uint32_t* gmax = (uint32_t*)s.head;
    k_nt_max<<<nvol, NT_THREADS, 0, ctx->stream>>>((const uint16_t*)volumes->dptr, (size_t)nz * N, gmax);
    EPID_CUDA(cudaGetLastError());
    EPID_SMEM_OPT_IN(ctx, k_nt_slices, s.smem);
    k_nt_slices<<<n, NT_THREADS, s.smem, ctx->stream>>>((const uint16_t*)volumes->dptr, nz, h, w, gmax, ufov_erode, (uint32_t*)s.ws,
                                                        (epid_nt_slice*)s.rows);
    ctx->launches += 2;
    return finish(ctx, results, s.rows, n * sizeof(epid_nt_slice), "tomographic slices");
}

extern "C" int32_t epid_nt_spheres(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, const struct epid_nt_sphere_in* spheres,
                                   int32_t nspheres, int32_t maxfun, int32_t maxiter, struct epid_nt_sphere* results) {
    EPID_REQUIRE(ctx && (spheres && results || nspheres == 0), EPID_ERR_INVALID, "NULL argument");
    int rc = nt_check(volumes, nz);
    if (rc != EPID_OK) return rc;
    EPID_REQUIRE(nspheres >= 0 && maxfun >= 0 && maxiter >= 0, EPID_ERR_INVALID, "negative count (nspheres %d, maxfun %d, maxiter %d)",
                 nspheres, maxfun, maxiter);
    const int nvol = volumes->n / nz;
    for (int i = 0; i < nspheres; i++)
        EPID_REQUIRE(spheres[i].volume >= 0 && spheres[i].volume < nvol, EPID_ERR_INVALID, "sphere %d: volume %d of %d", i,
                     spheres[i].volume, nvol);
    if (nspheres == 0) return EPID_OK;
    EPID_CUDA(cudaSetDevice(ctx->device));
    const size_t b_in = align256(nspheres * sizeof(epid_nt_sphere_in));
    if ((rc = ensure_scratch(ctx, b_in + align256(nspheres * sizeof(epid_nt_sphere)))) != EPID_OK) return rc;
    char* base = (char*)ctx->scratch;
    epid_nt_sphere_in* din = (epid_nt_sphere_in*)base;
    epid_nt_sphere* dres = (epid_nt_sphere*)(base + b_in);
    EPID_CUDA(cudaMemcpyAsync(din, spheres, nspheres * sizeof(epid_nt_sphere_in), cudaMemcpyHostToDevice, ctx->stream));
    k_nt_spheres<<<nspheres, NT_SPHERE_THREADS, 0, ctx->stream>>>((const uint16_t*)volumes->dptr, nz, volumes->h, volumes->w, din, maxfun,
                                                                  maxiter, dres);
    ctx->launches += 1;
    return finish(ctx, results, dres, nspheres * sizeof(epid_nt_sphere), "tomographic sphere search");
}
