// Block-cooperative scipy.signal.find_peaks on one fp64 profile (device code, one CTA per profile).
//
// Reproduces, stage for stage, what pylinac.core.profile.find_peaks (core/profile.py:2545-2623) obtains from
// scipy.signal.find_peaks(x, height, distance, prominence, width, rel_height)   (scipy/signal/_peak_finding.py:
// _local_maxima_1d, _select_by_peak_distance, _peak_prominences, _peak_widths; restated in SURVEY.md appendix B):
//   local maxima (plateau midpoint) -> height >= hmin -> distance (highest first) -> prominences (wlen=None)
//   -> prominence >= pmin -> widths at rel_height -> width >= wmin -> keep the max_number largest by `peak_sort`,
//   returned left to right.
// All arithmetic is IEEE fp64 in the same operation order as the reference (built with -fmad=false), so indices, bases,
// prominences, width heights and interpolated positions are bit-exact.
// Ties are resolved in one fixed order: among equal heights in the distance stage, and among equal keys at the
// max_number cut, the right-most candidate ranks highest.  That is scipy's and the reference's result whenever
// numpy's argsort keeps tied elements in their original order; the default argsort kind does not promise that, and
// where it does not, the reference's result on tied inputs depends on the CPU it runs on.
#pragma once
#include "common.cuh"

namespace epid {

constexpr int PK_WALK = 64;      // samples per side a lane walks on its own per round (block_find_peaks, prominences)
#ifndef EPID_PK_MAXBLK
#define EPID_PK_MAXBLK 512
#endif
constexpr int PK_MAXBLK = EPID_PK_MAXBLK;   // 32-sample blocks of the prominence skip table (profiles of up to 16384 samples)
constexpr int PK_RANK_MAX = 768; // distance stage: order by rank counting up to this many candidates, bitonic network beyond
constexpr int PK_COOP = 32;      // unfinished walks in a warp after a round that the warp finishes cooperatively (32 = all)

struct PeakArgs {          // already parsed (= after _parse_peak_args, core/profile.py:2626-2649)
    double hmin;           // height threshold (may be -inf)
    int distance;          // ceil(distance); <= 1 disables the stage
    double pmin;           // required prominence; < 0: none
    double wmin;           // min width
    double rel_height;     // 1 - fwxm_height
    int max_number;        // <= 0: all
    int sort_by_height;    // peak_sort == 'peak_heights'
};

struct PeakWork {          // caller-provided arrays (shared or global), each of capacity `cap`
    int cap;
    int* idx;
    double* prom;
    int* lbase;
    int* rbase;
    double* width_height;
    double* lip;
    double* rip;
    // scratch
    int* flag;             // cap
    double* skey;          // cap2 = next pow2 >= cap
    int* sidx;             // cap2
    int* s_small;          // >= blockDim.x + 8 ints
};

__device__ __forceinline__ bool key_less(double ka, int ia, double kb, int ib) { return ka < kb || (ka == kb && ia < ib); }

// ascending bitonic sort of (key, idx) pairs, m = power of two, all threads of the block participate
__device__ inline void block_bitonic_sort(double* key, int* idx, int m) {
    for (int k = 2; k <= m; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < m; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const bool up = (i & k) == 0;
                    const double ka = key[i], kb = key[l];
                    const int ia = idx[i], ib = idx[l];
                    const bool sw = up ? key_less(kb, ib, ka, ia) : key_less(ka, ia, kb, ib);
                    if (sw) {
                        key[i] = kb; key[l] = ka;
                        idx[i] = ib; idx[l] = ia;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// Order-preserving compaction of entries with flag != 0: chunks of blockDim.x entries, ballot + warp totals for the output
// positions; every source of a chunk is in registers before the first write (destinations never pass their sources).
__device__ inline int compact_by_flag(PeakWork& w, int count, bool have_props) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    __syncthreads();
    int out = 0;
    for (int base = 0; base < count; base += nt) {
        const int i = base + tid;
        const bool keep = i < count && w.flag[i] != 0;
        int idx = 0, lb = 0, rb = 0;
        double prom = 0, wh = 0, lip = 0, rip = 0;
        if (keep) {
            idx = w.idx[i];
            if (have_props) { prom = w.prom[i]; lb = w.lbase[i]; rb = w.rbase[i]; wh = w.width_height[i]; lip = w.lip[i]; rip = w.rip[i]; }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) w.s_small[1 + wid] = __popc(bal);
        __syncthreads();
        int woff = 0, total = 0;
        for (int k = 0; k < nw; k++) { const int c = w.s_small[1 + k]; if (k < wid) woff += c; total += c; }
        __syncthreads();
        if (keep) {
            const int o = out + woff + __popc(bal & ((1u << lane) - 1u));
            w.idx[o] = idx;
            if (have_props) { w.prom[o] = prom; w.lbase[o] = lb; w.rbase[o] = rb; w.width_height[o] = wh; w.lip[o] = lip; w.rip[o] = rip; }
        }
        out += total;
    }
    __syncthreads();
    return out;
}

// returns the number of peaks (>= 0) or -1 if the capacity was exceeded
__device__ inline int block_find_peaks(const double* __restrict__ x, int n, const PeakArgs& a, PeakWork& w) {
    const int tid = threadIdx.x, nt = blockDim.x;
    // ---- 1. local maxima + height filter, ordered.  Every warp owns one contiguous segment of the profile and sweeps it 32 samples at a
    // time (coalesced loads); a plateau is reported by its first sample (x[i-1] < x[i], look ahead over the equal samples, then a strictly
    // lower one) at its midpoint, exactly like _local_maxima_1d.  Pass 0 counts per warp, the warp totals are scanned, pass 1 writes.
    {
        const int lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
        const int span = n - 2;                                   // candidates i = 1 .. n - 2
        const int seg = span > 0 ? ((span + nw - 1) / nw + 31) / 32 * 32 : 0;
        const int i0 = 1 + wid * seg, i1 = min(n - 1, i0 + seg);
        int woff = 0;
        for (int pass = 0; pass < 2; pass++) {
            int o = woff;
            for (int b0 = i0; b0 < i1; b0 += 32) {
                const int i = b0 + lane;
                bool pk = false;
                int p = 0;
                if (i < i1) {
                    const double xi = x[i];
                    if (x[i - 1] < xi) {
                        int ahead = i + 1;
                        while (ahead < n - 1 && x[ahead] == xi) ahead++;
                        if (x[ahead] < xi) {
                            p = (i + ahead - 1) / 2;
                            pk = x[p] >= a.hmin;
                        }
                    }
                }
                const unsigned bal = __ballot_sync(0xffffffffu, pk);
                if (pass == 1 && pk) w.idx[o + __popc(bal & ((1u << lane) - 1u))] = p;
                o += __popc(bal);
            }
            if (pass == 0) {
                if (lane == 0) w.s_small[1 + wid] = o;
                __syncthreads();
                int total = 0;
                for (int k = 0; k < nw; k++) { const int c = w.s_small[1 + k]; if (k < wid) woff += c; total += c; }
                __syncthreads();
                if (tid == 0) w.s_small[0] = total;
                if (total > w.cap) return -1;
            }
        }
    }
    __syncthreads();
    int count = w.s_small[0];
    __syncthreads();
    if (count == 0) return 0;

    // ---- 2. distance
    if (a.distance > 1 && count > 1) {
        int m = 1;
        while (m < count) m <<= 1;
        for (int i = tid; i < m; i += nt) {
            if (i < count) { w.skey[i] = x[w.idx[i]]; w.sidx[i] = i; }
            else { w.skey[i] = __longlong_as_double(0x7ff0000000000000LL); w.sidx[i] = i; }  // +inf padding sorts last
            if (i < count) w.flag[i] = 1;
        }
        __syncthreads();
        // priority of every candidate = its rank in the ascending (height, position) order (a strict total order: among equal heights
        // the right-most candidate has the higher priority, as in _select_by_peak_distance), kept in w.lbase (free until stage 3)
        int* rank = w.lbase;
        if (count <= PK_RANK_MAX) {
            // by counting: rank = number of entries that sort before this one.  One barrier instead of the ~log2(m)^2 / 2 of the bitonic
            // network; every thread streams the same keys (broadcast loads).
            for (int i = tid; i < count; i += nt) {
                const double ki = w.skey[i];
                int r = 0;
#pragma unroll 4
                for (int j = 0; j < count; j++) r += key_less(w.skey[j], j, ki, i) ? 1 : 0;
                rank[i] = r;
            }
        } else {
            block_bitonic_sort(w.skey, w.sidx, m);
            for (int r = tid; r < count; r += nt) rank[w.sidx[r]] = r;
        }
        // scipy visits the candidates from the highest priority down and, for each one still kept, drops every neighbour closer than
        // `distance`: the lexicographically first maximal independent set.  The same set in parallel rounds: an undecided candidate
        // with a kept neighbour is dropped; one with no undecided neighbour of higher priority is kept; the others wait.  The highest
        // undecided candidate is settled every round, typically all of them within a few rounds.
        int* cur = w.flag;      // 2 undecided, 1 kept, 0 dropped
        int* nxt = w.rbase;     // (free until stage 3)
        for (int i = tid; i < count; i += nt) cur[i] = 2;
        __syncthreads();
        while (true) {
            bool waiting = false;
            for (int i = tid; i < count; i += nt) {
                int st = cur[i];
                if (st == 2) {
                    const int pi = w.idx[i], ri = rank[i];
                    bool has_kept = false, blocked = false;
                    for (int k = i - 1; k >= 0 && pi - w.idx[k] < a.distance; k--) {
                        const int sk = cur[k];
                        if (sk == 1) { has_kept = true; break; }
                        if (sk == 2 && rank[k] > ri) { blocked = true; break; }
                    }
                    if (!has_kept && !blocked) {
                        for (int k = i + 1; k < count && w.idx[k] - pi < a.distance; k++) {
                            const int sk = cur[k];
                            if (sk == 1) { has_kept = true; break; }
                            if (sk == 2 && rank[k] > ri) { blocked = true; break; }
                        }
                    }
                    st = has_kept ? 0 : (blocked ? 2 : 1);
                    waiting = waiting || st == 2;
                }
                nxt[i] = st;
            }
            const int more = __syncthreads_or(waiting ? 1 : 0);
            int* t = cur; cur = nxt; nxt = t;
            if (!more) break;
        }
        if (cur != w.flag) {
            for (int i = tid; i < count; i += nt) w.flag[i] = cur[i];
        }
        count = compact_by_flag(w, count, false);
    }

    // ---- 3. prominences (wlen = None): for every peak the minimum between it and the nearest HIGHER sample on either side (or the
    // end of the profile); among equal minima the sample closest to the peak is the base (scipy walks outwards and updates on "<").
    // Profiles of up to 32 * PK_MAXBLK samples: a table of 32-sample blocks (maximum, minimum, offsets of the first / last
    // occurrence of the minimum) lets a walk skip every block that holds no higher sample -- <= 32 + n / 32 + 32 steps instead of a
    // walk across the profile (the dominant peaks), with the same minima and bases.  Longer profiles: per-lane walks in rounds,
    // finished warp-cooperatively.
    __shared__ double s_bmax[PK_MAXBLK], s_bmin[PK_MAXBLK];
    __shared__ unsigned short s_bpos[PK_MAXBLK];           // first | last << 8: offsets of the block minimum
    const bool have_tab = n <= 32 * PK_MAXBLK;
    if (have_tab) {
        const int lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
        const int nblk = (n + 31) >> 5;
        __syncthreads();
        for (int b = wid; b < nblk; b += nw) {
            const int k = (b << 5) + lane;
            const bool in = k < n;
            const double v = in ? x[k] : 0.0;
            double vmax = in ? v : -__longlong_as_double(0x7ff0000000000000LL);
            double vmin = in ? v : __longlong_as_double(0x7ff0000000000000LL);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                vmax = fmax(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
                vmin = fmin(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
            }
            const unsigned eq = __ballot_sync(0xffffffffu, in && v == vmin);
            if (lane == 0) {
                s_bmax[b] = vmax;
                s_bmin[b] = vmin;
                s_bpos[b] = (unsigned short)((__ffs(eq) - 1) | ((31 - __clz(eq)) << 8));
            }
        }
        __syncthreads();
        for (int i = tid; i < count; i += nt) {
            const int p = w.idx[i];
            const double xp = x[p];
            const int pb_ = p >> 5;
            // left: own block downwards (fixed trip count, the loads do not depend on the running state), then whole blocks
            double lmin = xp;
            int lb = p;
            bool stop = false;
            for (int k = p; k >= (pb_ << 5); k--) {
                const double v = x[k];
                if (!stop) {
                    if (v > xp) stop = true;
                    else if (v < lmin) { lmin = v; lb = k; }
                }
            }
            for (int b = pb_ - 1; b >= 0 && !stop; b--) {
                if (s_bmax[b] > xp) {
                    for (int k = (b << 5) + 31; k >= (b << 5); k--) {
                        const double v = x[k];
                        if (!stop) {
                            if (v > xp) stop = true;
                            else if (v < lmin) { lmin = v; lb = k; }
                        }
                    }
                } else if (s_bmin[b] < lmin) {
                    lmin = s_bmin[b];
                    lb = (b << 5) + (s_bpos[b] >> 8);
                }
            }
            // right
            double rmin = xp;
            int rb = p;
            stop = false;
            const int own_end = min(n - 1, (pb_ << 5) + 31);
            for (int k = p; k <= own_end; k++) {
                const double v = x[k];
                if (!stop) {
                    if (v > xp) stop = true;
                    else if (v < rmin) { rmin = v; rb = k; }
                }
            }
            for (int b = pb_ + 1; b < nblk && !stop; b++) {
                if (s_bmax[b] > xp) {
                    const int e = min(n - 1, (b << 5) + 31);
                    for (int k = b << 5; k <= e; k++) {
                        const double v = x[k];
                        if (!stop) {
                            if (v > xp) stop = true;
                            else if (v < rmin) { rmin = v; rb = k; }
                        }
                    }
                } else if (s_bmin[b] < rmin) {
                    rmin = s_bmin[b];
                    rb = (b << 5) + (s_bpos[b] & 0xff);
                }
            }
            w.prom[i] = xp - fmax(lmin, rmin);
            w.lbase[i] = lb;
            w.rbase[i] = rb;
        }
    } else
    for (int base = 0; base < count; base += nt) {
        const int i = base + tid;
        const bool act = i < count;
        const int p = act ? w.idx[i] : 0;
        const double xp = act ? x[p] : 0.0;
        int kl = p, lb = p, kr = p, rb = p;
        double lmin = xp, rmin = xp;
        bool runl = act, runr = act;
        const int lane = tid & 31;
        while (true) {
            if (runl) {
                int steps = 0;
                while (kl >= 0 && x[kl] <= xp && steps < PK_WALK) { if (x[kl] < lmin) { lmin = x[kl]; lb = kl; } kl--; steps++; }
                runl = kl >= 0 && x[kl] <= xp;
            }
            if (runr) {
                int steps = 0;
                while (kr <= n - 1 && x[kr] <= xp && steps < PK_WALK) { if (x[kr] < rmin) { rmin = x[kr]; rb = kr; } kr++; steps++; }
                runr = kr <= n - 1 && x[kr] <= xp;
            }
            const unsigned pl = __ballot_sync(0xffffffffu, runl), pr = __ballot_sync(0xffffffffu, runr);
            if ((pl | pr) == 0) break;
            if (__popc(pl) + __popc(pr) > PK_COOP) continue;      // still many walkers: another round of per-lane walking
#pragma unroll 1
            for (int side = 0; side < 2; side++) {
                unsigned pend = side == 0 ? pl : pr;
                while (pend) {
                    const int src = __ffs(pend) - 1;
                    pend &= pend - 1;
                    int k0 = __shfl_sync(0xffffffffu, side == 0 ? kl : kr, src);
                    const double xps = __shfl_sync(0xffffffffu, xp, src);
                    double mn = __shfl_sync(0xffffffffu, side == 0 ? lmin : rmin, src);
                    int mb = __shfl_sync(0xffffffffu, side == 0 ? lb : rb, src);
                    while (true) {
                        const int kk = side == 0 ? k0 - lane : k0 + lane;
                        const bool inb = kk >= 0 && kk <= n - 1;
                        const double v = inb ? x[kk] : 0.0;
                        const bool stop = !(inb && v <= xps);
                        const unsigned sm = __ballot_sync(0xffffffffu, stop);
                        const int nvalid = sm ? __ffs(sm) - 1 : 32;
                        // minimum over the lanes inside the walk, the lowest lane (= closest sample) among equals
                        double bv = lane < nvalid ? v : __longlong_as_double(0x7ff0000000000000LL);
                        int bl = lane;
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) {
                            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                            const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
                            if (ov < bv || (ov == bv && ol < bl)) { bv = ov; bl = ol; }
                        }
                        if (nvalid > 0 && bv < mn) { mn = bv; mb = side == 0 ? k0 - bl : k0 + bl; }
                        if (sm) break;
                        k0 += side == 0 ? -32 : 32;
                    }
                    if (lane == src) { if (side == 0) { lmin = mn; lb = mb; } else { rmin = mn; rb = mb; } }
                }
            }
            break;
        }
        if (act) {
            w.prom[i] = xp - fmax(lmin, rmin);
            w.lbase[i] = lb;
            w.rbase[i] = rb;
        }
    }
    __syncthreads();
    // ---- 4/5. widths at rel_height (independent per peak).  The walk from the peak down to the evaluation height skips whole 32-sample
    // blocks whose minimum is still above that height (same table as the prominences): the dominant peak of a field profile would
    // otherwise walk thousands of samples in one thread.  When no minimum width is requested the widths cannot remove a peak, so they
    // are evaluated after the selection below, for the survivors only.
    auto widths = [&](int cnt, bool set_flags) {
        for (int i = tid; i < cnt; i += nt) {
            const int p = w.idx[i];
            const double h = x[p] - w.prom[i] * a.rel_height;
            const int imin = w.lbase[i], imax = w.rbase[i];
            int k = p;
            if (have_tab) {
                const int lim = max(imin, (p >> 5) << 5);
                while (lim < k && h < x[k]) k--;
                if (imin < k && h < x[k]) {                       // at the first sample of the peak's block, still above h
                    int b = (p >> 5) - 1;
                    while (b >= 0 && s_bmin[b] > h && (b << 5) > imin) b--;
                    k = ((b + 1) << 5) - 1;
                }
            }
            while (imin < k && h < x[k]) k--;
            double l = (double)k;
            if (x[k] < h) l += (h - x[k]) / (x[k + 1] - x[k]);
            k = p;
            if (have_tab) {
                const int lim = min(imax, ((p >> 5) << 5) + 31);
                while (k < lim && h < x[k]) k++;
                if (k < imax && h < x[k]) {                       // at the last sample of the peak's block, still above h
                    const int nblk = (n + 31) >> 5;
                    int b = (p >> 5) + 1;
                    while (b < nblk && s_bmin[b] > h && (b << 5) + 31 < imax) b++;
                    k = b << 5;
                }
            }
            while (k < imax && h < x[k]) k++;
            double r = (double)k;
            if (x[k] < h) r -= (h - x[k]) / (x[k - 1] - x[k]);
            w.width_height[i] = h;
            w.lip[i] = l;
            w.rip[i] = r;
            if (set_flags) w.flag[i] = ((a.pmin < 0 || w.prom[i] >= a.pmin) && (a.wmin <= r - l)) ? 1 : 0;
        }
    };
    const bool widths_first = a.wmin > 0.0;
    if (widths_first) widths(count, true);
    else for (int i = tid; i < count; i += nt) w.flag[i] = (a.pmin < 0 || w.prom[i] >= a.pmin) ? 1 : 0;
    count = compact_by_flag(w, count, true);
    if (count == 0) return 0;

    // ---- 6. keep the max_number largest by the sort key, left to right (core/profile.py:2615-2623)
    if (a.max_number == 1 && count > 1) {
        // the single largest entry by (key, position): what the last element of the ascending sort below would be
        const int lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
        double bk = -__longlong_as_double(0x7ff0000000000000LL);
        int bi = -1;
        for (int i = tid; i < count; i += nt) {
            const double k = a.sort_by_height ? x[w.idx[i]] : w.prom[i];
            if (bi < 0 || key_less(bk, bi, k, i)) { bk = k; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ok = __shfl_xor_sync(0xffffffffu, bk, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || key_less(bk, bi, ok, oi))) { bk = ok; bi = oi; }
        }
        __syncthreads();
        if (lane == 0) { w.s_small[1 + 3 * wid] = __double2hiint(bk); w.s_small[2 + 3 * wid] = __double2loint(bk); w.s_small[3 + 3 * wid] = bi; }
        __syncthreads();
        if (tid == 0) {
            double gk = 0;
            int gi = -1;
            for (int k = 0; k < nw; k++) {
                const int oi = w.s_small[3 + 3 * k];
                const double ok = __hiloint2double(w.s_small[1 + 3 * k], w.s_small[2 + 3 * k]);
                if (oi >= 0 && (gi < 0 || key_less(gk, gi, ok, oi))) { gk = ok; gi = oi; }
            }
            w.s_small[0] = gi;
        }
        __syncthreads();
        const int win = w.s_small[0];
        __syncthreads();
        for (int i = tid; i < count; i += nt) w.flag[i] = i == win ? 1 : 0;
        count = compact_by_flag(w, count, true);
    } else if (a.max_number > 0 && count > a.max_number) {
        int m = 1;
        while (m < count) m <<= 1;
        for (int i = tid; i < m; i += nt) {
            if (i < count) { w.skey[i] = a.sort_by_height ? x[w.idx[i]] : w.prom[i]; w.sidx[i] = i; w.flag[i] = 0; }
            else { w.skey[i] = __longlong_as_double(0x7ff0000000000000LL); w.sidx[i] = i; }
        }
        __syncthreads();
        block_bitonic_sort(w.skey, w.sidx, m);
        for (int i = tid; i < a.max_number; i += nt) w.flag[w.sidx[count - 1 - i]] = 1;
        count = compact_by_flag(w, count, true);
    }
    if (!widths_first) {
        widths(count, false);
        __syncthreads();
    }
    return count;
}

}  // namespace epid
