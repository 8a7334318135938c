// Runs epid::block_find_peaks (pylinac_b200/csrc/peaks.cuh) on its own, one CTA per run over a ragged batch of profiles, for
// tests/test_gpu_find_peaks.py.  The block size is chosen at run time; compile with the library's flags (-fmad=false keeps the fp64
// arithmetic in scipy's rounding), once as is and once with -DEPID_PK_MAXBLK=2 (the skip-table size of the PicketFence units).
//
//   peaks_harness <in.bin> <out.bin> <block>
//
// in (little-endian): int32 nruns, int64 nx, then per-run columns
//   int64 off[nruns]  int32 n[nruns]  int32 cap[nruns]  int32 distance[nruns]  int32 max_number[nruns]  int32 sort_by_height[nruns]
//   f64 hmin[nruns]  f64 pmin[nruns]  f64 wmin[nruns]  f64 rel_height[nruns],  then f64 x[nx]  (run r reads x[off[r] .. off[r] + n[r]))
// out: int32 count[nruns] (-1: more local maxima above hmin than cap), then for every run with count c > 0, in run order:
//   int32 idx[c]  int32 left_base[c]  int32 right_base[c]  f64 prominence[c]  f64 width_height[c]  f64 left_ip[c]  f64 right_ip[c]
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "peaks.cuh"

using namespace epid;

struct Run {
    long long off, slot, slot2;   // profile offset, offset of the run's cap-sized and cap2-sized work arrays
    int n, cap;
    PeakArgs a;
};

struct Work {
    int *idx, *lb, *rb, *flag, *sidx;
    double *prom, *wh, *lip, *rip, *skey;
};

template <int MAXT>
__global__ void __launch_bounds__(MAXT) k_peaks(const double* __restrict__ x, const Run* __restrict__ runs, Work g, int* count) {
    extern __shared__ int s_small[];                      // blockDim.x + 8 ints
    const Run r = runs[blockIdx.x];
    PeakWork w;
    w.cap = r.cap;
    w.idx = g.idx + r.slot; w.prom = g.prom + r.slot; w.lbase = g.lb + r.slot; w.rbase = g.rb + r.slot;
    w.width_height = g.wh + r.slot; w.lip = g.lip + r.slot; w.rip = g.rip + r.slot; w.flag = g.flag + r.slot;
    w.skey = g.skey + r.slot2; w.sidx = g.sidx + r.slot2;
    w.s_small = s_small;
    const int c = block_find_peaks(x + r.off, r.n, r.a, w);
    if (threadIdx.x == 0) count[blockIdx.x] = c;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
            return 1;                                                                              \
        }                                                                                          \
    } while (0)

template <class T>
static bool rd(FILE* f, T* p, size_t k) { return fread(p, sizeof(T), k, f) == k; }

template <class T>
static T* dalloc(size_t k) {
    T* p = nullptr;
    return cudaMalloc(&p, sizeof(T) * (k ? k : 1)) == cudaSuccess ? p : nullptr;
}

int main(int argc, char** argv) {
    if (argc != 4) { fprintf(stderr, "usage: %s in.bin out.bin block\n", argv[0]); return 2; }
    const int block = atoi(argv[3]);
    if (block < 32 || block > 1024 || block % 32) { fprintf(stderr, "block must be a multiple of 32 in [32, 1024]\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror(argv[1]); return 2; }
    int32_t nruns = 0;
    int64_t nx = 0;
    bool ok = rd(f, &nruns, 1) && rd(f, &nx, 1) && nruns >= 0 && nx >= 0;
    std::vector<int64_t> off(nruns);
    std::vector<int32_t> n(nruns), cap(nruns), dist(nruns), maxn(nruns), sbh(nruns);
    std::vector<double> hmin(nruns), pmin(nruns), wmin(nruns), relh(nruns), x(nx);
    ok = ok && rd(f, off.data(), nruns) && rd(f, n.data(), nruns) && rd(f, cap.data(), nruns) && rd(f, dist.data(), nruns) &&
         rd(f, maxn.data(), nruns) && rd(f, sbh.data(), nruns) && rd(f, hmin.data(), nruns) && rd(f, pmin.data(), nruns) &&
         rd(f, wmin.data(), nruns) && rd(f, relh.data(), nruns) && rd(f, x.data(), nx);
    fclose(f);
    if (!ok) { fprintf(stderr, "%s: truncated input\n", argv[1]); return 2; }

    std::vector<Run> runs(nruns);
    long long slots = 0, slots2 = 0;
    for (int r = 0; r < nruns; r++) {
        if (n[r] < 1 || off[r] < 0 || off[r] + n[r] > nx || cap[r] < 0) { fprintf(stderr, "run %d out of range\n", r); return 2; }
        int cap2 = 1;
        while (cap2 < cap[r]) cap2 <<= 1;
        Run& u = runs[r];
        u.off = off[r]; u.slot = slots; u.slot2 = slots2; u.n = n[r]; u.cap = cap[r];
        u.a.hmin = hmin[r]; u.a.distance = dist[r]; u.a.pmin = pmin[r]; u.a.wmin = wmin[r]; u.a.rel_height = relh[r];
        u.a.max_number = maxn[r]; u.a.sort_by_height = sbh[r];
        slots += cap[r];
        slots2 += cap2;
    }

    double* d_x = dalloc<double>(nx);
    Run* d_runs = dalloc<Run>(nruns);
    int* d_count = dalloc<int>(nruns);
    Work g;
    g.idx = dalloc<int>(slots); g.lb = dalloc<int>(slots); g.rb = dalloc<int>(slots); g.flag = dalloc<int>(slots);
    g.prom = dalloc<double>(slots); g.wh = dalloc<double>(slots); g.lip = dalloc<double>(slots); g.rip = dalloc<double>(slots);
    g.sidx = dalloc<int>(slots2); g.skey = dalloc<double>(slots2);
    if (!d_x || !d_runs || !d_count || !g.idx || !g.lb || !g.rb || !g.flag || !g.prom || !g.wh || !g.lip || !g.rip || !g.sidx || !g.skey) {
        fprintf(stderr, "cudaMalloc failed (%lld + %lld work slots)\n", slots, slots2);
        return 1;
    }
    CK(cudaMemcpy(d_x, x.data(), sizeof(double) * nx, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_runs, runs.data(), sizeof(Run) * nruns, cudaMemcpyHostToDevice));
    if (nruns > 0) {
        const size_t smem = sizeof(int) * (block + 8);
        if (block <= 256) k_peaks<256><<<nruns, block, smem>>>(d_x, d_runs, g, d_count);
        else k_peaks<1024><<<nruns, block, smem>>>(d_x, d_runs, g, d_count);
        CK(cudaGetLastError());
    }
    CK(cudaDeviceSynchronize());

    std::vector<int> count(nruns), hi, hl, hr;
    std::vector<double> hp, hw, hli, hri;
    CK(cudaMemcpy(count.data(), d_count, sizeof(int) * nruns, cudaMemcpyDeviceToHost));
    FILE* o = fopen(argv[2], "wb");
    if (!o) { perror(argv[2]); return 2; }
    fwrite(count.data(), sizeof(int), nruns, o);
    for (int r = 0; r < nruns; r++) {
        const int c = count[r];
        if (c <= 0) continue;
        if (c > cap[r]) { fprintf(stderr, "run %d: count %d above cap %d\n", r, c, cap[r]); fclose(o); return 1; }
        hi.resize(c); hl.resize(c); hr.resize(c); hp.resize(c); hw.resize(c); hli.resize(c); hri.resize(c);
        const long long s = runs[r].slot;
        CK(cudaMemcpy(hi.data(), g.idx + s, sizeof(int) * c, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hl.data(), g.lb + s, sizeof(int) * c, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hr.data(), g.rb + s, sizeof(int) * c, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hp.data(), g.prom + s, sizeof(double) * c, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hw.data(), g.wh + s, sizeof(double) * c, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hli.data(), g.lip + s, sizeof(double) * c, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hri.data(), g.rip + s, sizeof(double) * c, cudaMemcpyDeviceToHost));
        fwrite(hi.data(), sizeof(int), c, o); fwrite(hl.data(), sizeof(int), c, o); fwrite(hr.data(), sizeof(int), c, o);
        fwrite(hp.data(), sizeof(double), c, o); fwrite(hw.data(), sizeof(double), c, o);
        fwrite(hli.data(), sizeof(double), c, o); fwrite(hri.data(), sizeof(double), c, o);
    }
    const bool wok = fclose(o) == 0;
    cudaFree(d_x); cudaFree(d_runs); cudaFree(d_count);
    cudaFree(g.idx); cudaFree(g.lb); cudaFree(g.rb); cudaFree(g.flag); cudaFree(g.prom); cudaFree(g.wh); cudaFree(g.lip); cudaFree(g.rip);
    cudaFree(g.sidx); cudaFree(g.skey);
    if (!wok) { fprintf(stderr, "%s: write failed\n", argv[2]); return 1; }
    printf("%d runs, block %d, PK_MAXBLK %d\n", nruns, block, PK_MAXBLK);
    return 0;
}
