// Varian XIM pixel decode: XIM._parse_lookup_table / _parse_compressed_bytes / _get_diffs (core/image.py:1186-1309) for a batch.
//
// The reference's row loop is the raster recurrence, modulo 2^(8 bpp):
//     v[i] = d[i] + v[i-1] + v[i-W] - v[i-W-1]       (i >= W+1; v[0..W] are the raw int32 head, truncated)
// With e[i] = v[i] - v[i-W] this is e[i] = e[i-1] + d[i] (e[W] = v[W] - v[0]) and v[i] = v[i-W] + e[i]: a flat inclusive scan of
// the diffs followed by a per-column inclusive scan of e.  Diff j (raster index W+1+j) has the 2-bit lookup code j; its width is
// 1 << code bytes and its byte offset is the prefix sum of the widths, so a tile finds its compressed bytes from a scan of the
// per-tile byte totals, which depend on the lookup codes alone.
//
// Launch sequence for the whole batch (frames may have different compressed sizes):
//   k_xim_tile_bytes   per (tile, frame): byte total of the tile's diffs; first code 3 anywhere in the table (atomicMin)
//   k_xim_scan         per frame: exclusive scan of the tile byte totals (+ the frame's total)
//   k_xim_status       per frame: ok / code 3 / buffer too short, in the order the reference raises them
//   k_xim_tile_diffs   per (tile, frame): one cp.async.bulk copy of the tile's byte range into shared memory, gather the diffs,
//                      block scan -> tile-local inclusive scan of d (stored) and the tile's sum
//   k_xim_scan         per frame: exclusive scan of the tile sums (the flat scan's carry into each tile)
//   k_xim_columns      per (column, frame): v = raw head + running sum of e down the column, range check for U16 output
#include "common.cuh"
#include "tma.cuh"

namespace epid {
namespace {

constexpr int XT_THREADS = 256;
constexpr int XT_PER_THREAD = 16;                         // codes per thread = 4 lookup bytes = one 32-bit word
constexpr int XT_TILE = XT_THREADS * XT_PER_THREAD;       // diffs per tile
constexpr int XT_SMEM = XT_TILE * 4 + 32;                 // widest tile (all 4-byte diffs) + alignment slack at both ends

struct XimFrame {
    int64_t lut_off, lut_size, pix_off, pix_size;          // byte offsets / sizes inside the arena
};

__device__ __forceinline__ uint32_t lut_word(const uint8_t* arena, const XimFrame& fr, int64_t j0) {
    // the 16 codes j0 .. j0+15 (j0 % 16 == 0); codes past the end of the table read as 0 here and get width 0 from `ncodes`
    int64_t b = j0 >> 2;
    if (b + 4 <= fr.lut_size) return *reinterpret_cast<const uint32_t*>(arena + fr.lut_off + b);
    uint32_t w = 0;
    for (int k = 0; k < 4; k++)
        if (b + k < fr.lut_size) w |= (uint32_t)arena[fr.lut_off + b + k] << (8 * k);
    return w;
}

// width in bytes of code c of diff j (0 past the end of the table; code 3 is an error, counted as 0 so sums stay bounded)
__device__ __forceinline__ uint32_t code_width(uint32_t c, int64_t j, int64_t ncodes) {
    return (j < ncodes && c != 3u) ? (1u << c) : 0u;
}

template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* warp_tot, T* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    T incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        T u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        T s = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : T(0);
        T si = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            T u = __shfl_up_sync(0xffffffffu, si, o);
            if (lane >= o) si += u;
        }
        if (lane < (int)(blockDim.x >> 5)) warp_tot[lane] = si - s;
        if (lane == 31) *total = si;
    }
    __syncthreads();
    T r = warp_tot[wid] + incl - v;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(XT_THREADS) k_xim_tile_bytes(const uint8_t* __restrict__ arena, const XimFrame* __restrict__ frames,
                                                               int64_t D, int ntiles, uint64_t* __restrict__ tile_bytes,
                                                               unsigned long long* __restrict__ first3) {
    __shared__ uint64_t warp_tot[XT_THREADS / 32];
    __shared__ uint64_t total;
    const int f = blockIdx.y, t = blockIdx.x;
    const XimFrame fr = frames[f];
    const int64_t ncodes = fr.lut_size * 4;
    const int64_t j0 = (int64_t)t * XT_TILE + threadIdx.x * XT_PER_THREAD;
    uint32_t bytes = 0;
    int64_t bad = -1;
    if (j0 < D && j0 < ncodes) {
        const uint32_t w = lut_word(arena, fr, j0);
#pragma unroll
        for (int k = 0; k < XT_PER_THREAD; k++) {
            const int64_t j = j0 + k;
            const uint32_t c = (w >> (2 * k)) & 3u;
            if (j < D) bytes += code_width(c, j, ncodes);
            if (c == 3u && j < ncodes && bad < 0) bad = j;
        }
    }
    // the reference looks every run of the table up in LOOKUP_CONVERSION, including the padding after the last diff: the last
    // tile also scans the codes past D
    if (t == ntiles - 1) {
        const int64_t pad0 = ((D + 15) / 16) * 16;        // codes below pad0 belong to some thread's 16-code word above
        for (int64_t jw = pad0 + (int64_t)threadIdx.x * 16; jw < ncodes && bad < 0; jw += (int64_t)XT_THREADS * 16) {
            const uint32_t w = lut_word(arena, fr, jw);
            for (int k = 0; k < 16; k++)
                if (jw + k < ncodes && ((w >> (2 * k)) & 3u) == 3u) { bad = jw + k; break; }
        }
    }
    if (bad >= 0) atomicMin(first3 + f, (unsigned long long)bad);
    block_exclusive_scan<uint64_t>(bytes, warp_tot, &total);
    if (threadIdx.x == 0) tile_bytes[(size_t)f * ntiles + t] = total;
}

// per frame (one CTA): in[f][0..m) -> out[f][0..m] exclusive prefix sums, out[f][m] = total
__global__ void __launch_bounds__(1024) k_xim_scan(const uint64_t* __restrict__ in, int m, uint64_t* __restrict__ out) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t total;
    const int f = blockIdx.x;
    const uint64_t* src = in + (size_t)f * m;
    uint64_t* dst = out + (size_t)f * (m + 1);
    uint64_t carry = 0;
    for (int base = 0; base < m; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const uint64_t v = i < m ? src[i] : 0;
        const uint64_t ex = block_exclusive_scan<uint64_t>(v, warp_tot, &total);
        if (i < m) dst[i] = carry + ex;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) dst[m] = carry;
}

// per frame: the reference walks the runs of equal codes in order; a run that needs more bytes than are left raises ValueError
// (broadcast / view of a short slice), the first run of code 3 raises KeyError.  So "too short" wins exactly when the diffs
// before the first code 3 (or all diffs) need more bytes than the buffer holds past the raw head.
__global__ void k_xim_status(const uint8_t* __restrict__ arena, const XimFrame* __restrict__ frames, int n, int64_t D, int64_t head,
                             int ntiles, const uint64_t* __restrict__ byte_off, const unsigned long long* __restrict__ first3,
                             int32_t* __restrict__ status) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    const XimFrame fr = frames[f];
    const uint64_t* off = byte_off + (size_t)f * (ntiles + 1);
    const unsigned long long b3 = first3[f];
    const int64_t ncodes = fr.lut_size * 4;
    uint64_t need;
    if ((long long)b3 >= 0 && (int64_t)b3 < D) {
        const int64_t t = (int64_t)b3 / XT_TILE;
        need = off[t];
        for (int64_t j = t * XT_TILE; j < (int64_t)b3; j++) {
            const uint32_t c = (arena[fr.lut_off + (j >> 2)] >> (2 * (j & 3))) & 3u;
            need += code_width(c, j, ncodes);
        }
    } else {
        need = off[ntiles];
    }
    int32_t s = EPID_XIM_OK;
    if (fr.pix_size < head || (uint64_t)(fr.pix_size - head) < need) s = EPID_XIM_SHORT_BUFFER;
    else if (b3 != ~0ull) s = EPID_XIM_LOOKUP_CODE3;
    status[f] = s;
}

template <typename A>
__device__ __forceinline__ A sext_diff(const uint8_t* p, uint32_t width) {
    int32_t v;
    if (width == 1) v = (int8_t)p[0];
    else if (width == 2) v = (int16_t)(p[0] | (p[1] << 8));
    else if (width == 4) v = (int32_t)(p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24));
    else v = 0;
    return (A)(int64_t)v;
}

// E: storage type of the tile-local scan (bpp bytes); A: arithmetic type (32 or 64 bit, wraps like the output dtype)
template <typename E, typename A>
__global__ void __launch_bounds__(XT_THREADS) k_xim_tile_diffs(const uint8_t* __restrict__ arena, const XimFrame* __restrict__ frames,
                                                               int64_t D, int64_t W, size_t e_stride, int ntiles,
                                                               const uint64_t* __restrict__ byte_off, E* eloc, uint64_t* __restrict__ tile_sum) {
    __shared__ __align__(128) uint8_t buf[XT_SMEM];
    __shared__ __align__(8) uint64_t bar;
    __shared__ A warp_tot[XT_THREADS / 32];
    __shared__ A total;
    __shared__ uint32_t warp_tot32[XT_THREADS / 32];
    __shared__ uint32_t total32;
    const int f = blockIdx.y, t = blockIdx.x;
    const XimFrame fr = frames[f];
    const int64_t ncodes = fr.lut_size * 4;
    const int64_t head = 4 * (W + 1);
    const uint64_t* off = byte_off + (size_t)f * (ntiles + 1);
    const uint64_t tb0 = off[t], tb1 = off[t + 1];

    // the tile's byte range, clipped to the frame's pixel buffer (a short buffer is reported by k_xim_status; its tail reads 0)
    const uint8_t* slot = arena + fr.pix_off;
    const int64_t lo = head + (int64_t)tb0, hi = min(head + (int64_t)tb1, fr.pix_size);
    const uintptr_t a0 = (uintptr_t)(slot + lo) & ~(uintptr_t)15;
    const uintptr_t a1 = hi > lo ? (((uintptr_t)(slot + hi) + 15) & ~(uintptr_t)15) : a0;
    const uint32_t shift = (uint32_t)((uintptr_t)(slot + lo) - a0);
    const uint32_t nbytes = (uint32_t)(a1 - a0);
    const uint32_t bar_s = smem_u32(&bar);
    if (nbytes) {
        if (threadIdx.x == 0) {
            mbar_init(bar_s, 1);
            mbar_fence_init();
            mbar_expect_tx(bar_s, nbytes);
            tma_load_1d(smem_u32(buf), (const void*)a0, nbytes, bar_s);
        }
    }

    // codes of this thread's 16 diffs -> widths and the thread's byte offset inside the tile (overlaps the copy)
    const int64_t j0 = (int64_t)t * XT_TILE + threadIdx.x * XT_PER_THREAD;
    const uint32_t w = (j0 < D && j0 < ncodes) ? lut_word(arena, fr, j0) : 0u;
    uint32_t mybytes = 0;
#pragma unroll
    for (int k = 0; k < XT_PER_THREAD; k++)
        if (j0 + k < D) mybytes += code_width((w >> (2 * k)) & 3u, j0 + k, ncodes);
    uint32_t pos = block_exclusive_scan<uint32_t>(mybytes, warp_tot32, &total32);   // its __syncthreads orders mbar_init
    if (nbytes) mbar_wait(bar_s, 0);

    const int64_t avail = hi - lo;           // bytes of this tile actually present
    A run = 0;
    A vals[XT_PER_THREAD];
#pragma unroll
    for (int k = 0; k < XT_PER_THREAD; k++) {
        const int64_t j = j0 + k;
        A d = 0;
        if (j < D) {
            const uint32_t wd = code_width((w >> (2 * k)) & 3u, j, ncodes);
            if (wd && (int64_t)(pos + wd) <= avail) d = sext_diff<A>(buf + shift + pos, wd);
            pos += wd;
        }
        run += d;
        vals[k] = run;
    }
    const A ex = block_exclusive_scan<A>(run, warp_tot, &total);
    if (j0 < D) {
        E* dst = eloc + (size_t)f * e_stride + (W + 1 + j0);
#pragma unroll
        for (int k = 0; k < XT_PER_THREAD; k++)
            if (j0 + k < D) dst[k] = (E)(ex + vals[k]);
    }
    if (threadIdx.x == 0) tile_sum[(size_t)f * ntiles + t] = (uint64_t)total;
}

template <typename E>
__device__ __forceinline__ int64_t sext_e(uint64_t v) {
    if (sizeof(E) == 1) return (int8_t)v;
    if (sizeof(E) == 2) return (int16_t)v;
    if (sizeof(E) == 4) return (int32_t)v;
    return (int64_t)v;
}

// per (column, frame): v[0][c] = raw[c]; v[r][c] = v[r-1][c] + e[r][c], e = base + carry[tile] + tile-local scan.  O is the output
// dtype; U16 output checks every value of the reference's dtype (E, signed) against [0, 65535].
template <typename E, typename A, typename O, bool U16>
__global__ void __launch_bounds__(128) k_xim_columns(const uint8_t* __restrict__ arena, const XimFrame* __restrict__ frames, int64_t H,
                                                     int64_t W, int ntiles, const E* eloc, size_t e_frame_stride,
                                                     const uint64_t* __restrict__ carry, O* out, int32_t* __restrict__ status) {
    // eloc may alias out (same bytes, same thread): no __restrict__ on either
    const int f = blockIdx.y;
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= W) return;
    const XimFrame fr = frames[f];
    const uint8_t* slot = arena + fr.pix_off;
    auto raw = [&](int64_t k) -> A {
        if (4 * k + 4 > fr.pix_size) return A(0);
        const uint8_t* p = slot + 4 * k;
        return (A)(int64_t)(int32_t)(p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24));
    };
    const uint64_t* cf = carry + (size_t)f * (ntiles + 1);
    const E* ef = eloc + (size_t)f * e_frame_stride;
    O* of = out + (size_t)f * H * W;
    const A base = raw(W) - raw(0);
    A v = raw(c);
    bool bad = false;
    auto store = [&](int64_t i, A x) {
        const int64_t s = sext_e<E>((uint64_t)x);
        if (U16) {
            bad |= (s < 0 || s > 65535);
            of[i] = (O)(uint16_t)s;
        } else {
            of[i] = (O)s;
        }
    };
    store(c, v);
    for (int64_t r = 1; r < H; r++) {
        const int64_t i = r * W + c;
        if (i == W) v += base;              // raster index W: e = v[W] - v[0], the raw value
        else v += base + (A)cf[(i - W - 1) / XT_TILE] + (A)ef[i];
        store(i, v);
    }
    if (U16 && bad && status[f] == EPID_XIM_OK) status[f] = EPID_XIM_U16_RANGE;
}

// N: the reference's output dtype for this bpp
template <typename E, typename A, typename N>
int launch_decode(epid_ctx* ctx, const uint8_t* d_arena, const XimFrame* d_frames, int n, int64_t H, int64_t W, int ntiles,
                  const uint64_t* d_off, uint64_t* d_tsum, uint64_t* d_carry, E* eloc, size_t e_stride, epid_batch* out, int32_t* d_status) {
    const int64_t D = H * W - W - 1;
    k_xim_tile_diffs<E, A><<<dim3(ntiles, n), XT_THREADS, 0, ctx->stream>>>(d_arena, d_frames, D, W, e_stride, ntiles, d_off, eloc, d_tsum);
    k_xim_scan<<<n, 1024, 0, ctx->stream>>>(d_tsum, ntiles, d_carry);
    const dim3 cg((unsigned)((W + 127) / 128), n);
    if (out->dtype == EPID_U16)
        k_xim_columns<E, A, uint16_t, true><<<cg, 128, 0, ctx->stream>>>(d_arena, d_frames, H, W, ntiles, eloc, e_stride, d_carry,
                                                                        (uint16_t*)out->dptr, d_status);
    else
        k_xim_columns<E, A, N, false><<<cg, 128, 0, ctx->stream>>>(d_arena, d_frames, H, W, ntiles, eloc, e_stride, d_carry,
                                                                  (N*)out->dptr, d_status);
    ctx->launches += 3;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace
}  // namespace epid

using namespace epid;

extern "C" int32_t epid_xim_decode(epid_ctx* ctx, const void* arena, size_t arena_bytes, const int64_t* desc, int32_t n, int32_t h,
                                   int32_t w, int32_t bpp, int32_t dtype, int32_t* status, epid_batch** out) {
    EPID_REQUIRE(ctx && arena && desc && status && out, EPID_ERR_INVALID, "NULL argument");
    *out = nullptr;
    EPID_REQUIRE(n > 0 && n <= 65535, EPID_ERR_INVALID, "n = %d frames (1 .. 65535 per call)", n);
    EPID_REQUIRE(w > 0 && h > 1, EPID_ERR_INVALID, "XIM decode needs at least 2 rows (got %d x %d)", h, w);
    EPID_REQUIRE(bpp == 1 || bpp == 2 || bpp == 4 || bpp == 8, EPID_ERR_INVALID,
                 "The XIM image has an unsupported bytes per pixel value (%d)", bpp);
    const int natural = bpp == 8 ? EPID_I64 : bpp == 4 ? EPID_I32 : EPID_I16;
    EPID_REQUIRE(dtype == natural || dtype == EPID_U16, EPID_ERR_INVALID, "output dtype %d does not hold bpp %d pixels", dtype, bpp);
    EPID_REQUIRE(((uintptr_t)arena & 15) == 0, EPID_ERR_INVALID, "arena must be 16-byte aligned");
    for (int f = 0; f < n; f++) {
        const int64_t* d = desc + 4 * (size_t)f;
        EPID_REQUIRE(d[0] >= 0 && d[1] >= 0 && d[2] >= 0 && d[3] >= 0 && d[0] + d[1] <= (int64_t)arena_bytes &&
                         d[2] + d[3] <= (int64_t)arena_bytes && (d[0] & 15) == 0 && (d[2] & 15) == 0,
                     EPID_ERR_INVALID, "frame %d: descriptor outside the arena or not 16-byte aligned", f);
    }
    const int64_t H = h, W = w, D = H * W - W - 1;
    const int ntiles = D > 0 ? (int)((D + XT_TILE - 1) / XT_TILE) : 1;
    EPID_CUDA(cudaSetDevice(ctx->device));

    // scratch: arena | frame descriptors | first3 | tile bytes | byte offsets | tile sums | carries | status | tile-local scan
    const size_t e_size = (size_t)bpp;
    const bool e_in_out = dtype != EPID_U16 && e_size == dtype_size(dtype);
    const size_t arena_dev = align256((arena_bytes + 15) & ~(size_t)15) + 256;
    const size_t sz_fr = align256(sizeof(XimFrame) * n), sz_f3 = align256(8 * (size_t)n);
    const size_t sz_t = align256(8 * (size_t)n * ntiles), sz_o = align256(8 * (size_t)n * (ntiles + 1));
    const size_t sz_st = align256(4 * (size_t)n);
    const size_t sz_e = e_in_out ? 0 : align256(e_size * (size_t)n * H * W);
    const size_t total = arena_dev + sz_fr + sz_f3 + 2 * sz_t + 2 * sz_o + sz_st + sz_e;
    int rc = ensure_scratch(ctx, total);
    if (rc != EPID_OK) return rc;
    char* p = (char*)ctx->scratch;
    uint8_t* d_arena = (uint8_t*)p; p += arena_dev;
    XimFrame* d_frames = (XimFrame*)p; p += sz_fr;
    unsigned long long* d_first3 = (unsigned long long*)p; p += sz_f3;
    uint64_t* d_tbytes = (uint64_t*)p; p += sz_t;
    uint64_t* d_off = (uint64_t*)p; p += sz_o;
    uint64_t* d_tsum = (uint64_t*)p; p += sz_t;
    uint64_t* d_carry = (uint64_t*)p; p += sz_o;
    int32_t* d_status = (int32_t*)p; p += sz_st;
    void* d_e = sz_e ? (void*)p : nullptr;

    rc = epid_batch_alloc(ctx, dtype, n, h, w, out);
    if (rc != EPID_OK) return rc;
    epid_batch* b = *out;
    if (!d_e) d_e = b->dptr;
    auto fail = [&](cudaError_t e) {
        set_error("XIM decode: %s", cudaGetErrorString(e));
        epid_batch_free(b);
        *out = nullptr;
        return EPID_ERR_CUDA;
    };
    cudaStream_t s = ctx->stream;
    cudaError_t e = cudaMemcpyAsync(d_arena, arena, arena_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_frames, desc, sizeof(XimFrame) * n, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_first3, 0xff, 8 * (size_t)n, s);
    if (e != cudaSuccess) return fail(e);
    k_xim_tile_bytes<<<dim3(ntiles, n), XT_THREADS, 0, s>>>(d_arena, d_frames, D, ntiles, d_tbytes, d_first3);
    k_xim_scan<<<n, 1024, 0, s>>>(d_tbytes, ntiles, d_off);
    k_xim_status<<<(n + 127) / 128, 128, 0, s>>>(d_arena, d_frames, n, D, 4 * (W + 1), ntiles, d_off, d_first3, d_status);
    ctx->launches += 3;
    const size_t stride = (size_t)H * W;
    switch (bpp) {
        case 1: rc = launch_decode<uint8_t, uint32_t, int16_t>(ctx, d_arena, d_frames, n, H, W, ntiles, d_off, d_tsum, d_carry, (uint8_t*)d_e, stride, b, d_status); break;
        case 2: rc = launch_decode<uint16_t, uint32_t, int16_t>(ctx, d_arena, d_frames, n, H, W, ntiles, d_off, d_tsum, d_carry, (uint16_t*)d_e, stride, b, d_status); break;
        case 4: rc = launch_decode<uint32_t, uint32_t, int32_t>(ctx, d_arena, d_frames, n, H, W, ntiles, d_off, d_tsum, d_carry, (uint32_t*)d_e, stride, b, d_status); break;
        default: rc = launch_decode<uint64_t, uint64_t, int64_t>(ctx, d_arena, d_frames, n, H, W, ntiles, d_off, d_tsum, d_carry, (uint64_t*)d_e, stride, b, d_status); break;
    }
    if (rc != EPID_OK) {
        epid_batch_free(b);
        *out = nullptr;
        return rc;
    }
    e = cudaMemcpyAsync(status, d_status, 4 * (size_t)n, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(e);
    return EPID_OK;
}
