// Last stage of the batched PicketFence pipeline: one CTA per frame turns the per-window FWHM edges into the
// measurement table and the PFResult scalars.
//
// Reference semantics: leaf-row pruning by the median kiss count (picketfence.py:810-828), MLCValue.get_peak_positions /
// error / marker_lines (picketfence.py:1605-1628, 1701-1743), Picket.get_fit / dist2cax / skew (picketfence.py:1881-1923),
// aggregates (picketfence.py:439-562, 1313-1363, 1467-1469).
//
// Everything that scales with the number of measurements runs data-parallel: thread per (leaf, picket) pair for the table
// and the errors (the table index of a pair is its leaf row's offset plus a popcount over the row's validity mask), warp per
// picket for the line fits and the width statistics, block reductions for the aggregates.  The O(leaves) and O(pickets)
// bookkeeping (kiss-count median, row offsets, fit check, dist2cax / skew / picket spacing) runs on one warp.
#include "pf_common.cuh"

namespace epid {

constexpr int FIN_WARPS = FIN_THREADS / 32;
constexpr int FIN_LPL = (PF_L + 31) / 32;       // leaf slots per lane

// np.median of n non-negative doubles a[0..n) (shared memory) by the whole block: radix selection of the lower middle order
// statistic on the bit patterns (for non-negative doubles the unsigned order of the bits is the order of the values), up to eight
// 8-bit digits, warp-aggregated shared-memory histograms, stopping at the first digit whose bucket holds one value; the upper
// middle value is the same value if it occurs often enough, else the
// smallest larger one.  Thread 0 returns the median; every thread must call.
__device__ inline double block_median_nonneg_f64(const double* __restrict__ a, int n) {
    __shared__ uint32_t s_hist[256];
    __shared__ unsigned long long s_prefix, s_above;
    __shared__ uint32_t s_k, s_cle;
    const int tid = threadIdx.x, lane = tid & 31;
    auto keyat = [&](int i) { return (unsigned long long)__double_as_longlong(a[i]); };
    const int nround = (n + FIN_THREADS - 1) / FIN_THREADS * FIN_THREADS;      // every thread takes the same number of trips
    const int k1 = (n - 1) / 2, k2 = n / 2;
    unsigned long long prefix = 0, mask = 0;
    uint32_t k = (uint32_t)k1;
    for (int shift = 56; shift >= 0; shift -= 8) {
        s_hist[tid & 255] = 0;
        __syncthreads();
        for (int i = tid; i < nround; i += FIN_THREADS) {
            const unsigned long long kv = i < n ? keyat(i) : 0ull;
            const bool on = i < n && (kv & mask) == prefix;
            const uint32_t d = (uint32_t)(kv >> shift) & 255u;
            const unsigned m = __match_any_sync(0xffffffffu, on ? d : 256u);
            if (on && lane == __ffs(m) - 1) atomicAdd(&s_hist[d], (uint32_t)__popc(m));
        }
        __syncthreads();
        if (tid < 32) {
            uint32_t loc[8], sum = 0;
#pragma unroll
            for (int e = 0; e < 8; e++) { loc[e] = s_hist[tid * 8 + e]; sum += loc[e]; }
            uint32_t inc = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            uint32_t cum = inc - sum;
            if (k >= cum && k < inc) {      // exactly one lane
#pragma unroll
                for (int e = 0; e < 8; e++) {
                    if (k >= cum && k < cum + loc[e]) {
                        s_k = k - cum;
                        s_prefix = prefix | ((unsigned long long)(tid * 8 + e) << shift);
                        s_cle = loc[e];
                    }
                    cum += loc[e];
                }
            }
        }
        __syncthreads();
        prefix = s_prefix;
        k = s_k;
        mask |= 0xffull << shift;
        if (s_cle == 1u) {      // one value has this prefix: it is the order statistic, the lower digits need no more rounds
            __syncthreads();    // every thread has read s_prefix
            for (int i = tid; i < n; i += FIN_THREADS) {
                const unsigned long long kv = keyat(i);
                if ((kv & mask) == prefix) s_prefix = kv;
            }
            __syncthreads();
            prefix = s_prefix;
            break;
        }
    }
    // upper middle value
    if (tid == 0) { s_cle = 0; s_above = ~0ull; }
    __syncthreads();
    uint32_t c = 0;
    unsigned long long above = ~0ull;
    for (int i = tid; i < n; i += FIN_THREADS) {
        const unsigned long long kv = keyat(i);
        c += kv <= prefix ? 1u : 0u;
        if (kv > prefix && kv < above) above = kv;
    }
    c = __reduce_add_sync(0xffffffffu, c);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, above, o); above = t < above ? t : above; }
    if (lane == 0) { atomicAdd(&s_cle, c); atomicMin(&s_above, above); }
    __syncthreads();
    const double v1 = __longlong_as_double((long long)prefix);
    const double v2 = (s_cle >= (uint32_t)k2 + 1u) ? v1 : __longlong_as_double((long long)s_above);
    return (n & 1) ? v1 : (v1 + v2) / 2.0;
}

// 64 registers at 256 threads: four CTAs per SM, so a batch of up to 528 frames runs in one wave on 132 SMs
__global__ void __launch_bounds__(FIN_THREADS, 4)
k_pf_finalize(const PfConst* __restrict__ cc, PfFrame* fr, const PfWin* __restrict__ wins, epid_pf_summary* __restrict__ summ,
              epid_pf_meas* __restrict__ meas_all) {
    extern __shared__ double s_err[];                    // pow2(2 * meas_cap) doubles for the median of |errors|
    __shared__ int s_cnt[PF_L], s_off[PF_L], s_keep[PF_L], s_leafnum[PF_L];
    __shared__ uint32_t s_vmask[PF_L];
    __shared__ double s_upper[PF_L], s_centre[PF_L];
    __shared__ double s_fit[PF_P][2], s_offp[PF_P], s_srt[PF_P];
    __shared__ double s_cax, s_xmid;
    __shared__ int s_hist[PF_P + 1];                     // leaf rows per kiss count
    __shared__ int s_i[8];
    __shared__ double s_wbuf[FIN_WARPS][PF_L], s_wsort[FIN_WARPS][PF_L];
    __shared__ double s_rmax[FIN_WARPS];
    __shared__ int s_rarg[FIN_WARPS], s_rloc[FIN_WARPS], s_rpass[FIN_WARPS], s_rfail[FIN_WARPS];

    const int fi = blockIdx.x;
    const PfConst& c = *cc;
    PfFrame& f = fr[fi];
    epid_pf_summary& S = summ[fi];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int H = c.H, W = c.W;
    // every word of the row is defined, whatever the frame's fate: rows of different runs / pipelines compare equal byte for byte
    for (int k = tid; k < (int)(sizeof(epid_pf_summary) / 4); k += FIN_THREADS) reinterpret_cast<uint32_t*>(&S)[k] = 0u;
    if (tid <= PF_P) s_hist[tid] = 0;
    __syncthreads();
    if (tid == 0) {
        S.status = f.status;
        S.orientation = f.orientation;
        S.noise_median_passes = f.noise_passes;
        S.corner_inverted = f.corner_inverted;
        S.height = H;
        S.width = W;
        S.n_pickets = f.n_pickets;
        S.n_meas = 0;
        S.n_leaves_removed = 0;
        S.picket_spacing_px = f.spacing;
        // dist2cax (picketfence.py:1905-1923) / image.center (core/image.py:526-533, PFDicomImage.center :246-260)
        const int orient = f.orientation;
        s_cax = c.p.has_cax_override ? (orient == 0 ? c.p.cax_x_px : c.p.cax_y_px) : (orient == 0 ? (double)W : (double)H) / 2.0 - 0.5;
        s_xmid = rint((double)(orient == 0 ? H : W) / 2.0);
    }
    if (tid < PF_P) {
        S.picket_idx[tid] = tid < f.n_pickets ? f.picket_idx[tid] : 0;
        S.picket_val[tid] = tid < f.n_pickets ? f.picket_val[tid] : 0.0;
    }
    if (f.status != EPID_PF_OK) return;
    const int nl = f.n_inview, np = f.n_pickets;
    const int orient = f.orientation;
    const int npos = c.p.separate_leaves ? 2 : 1;
    const double dpmm = c.p.dpmm;
    const double spacing = f.spacing;
    const PfWin* wf = wins + (size_t)fi * PF_L * PF_P;
    const double n_axis_half = (orient == 0 ? (double)H : (double)W) / 2.0;
    const double ratio = c.p.leaf_analysis_width_ratio;
    // ---- kisses per leaf row, marker-line geometry of the row (picketfence.py:1725-1743)
    if (tid < np) s_offp[tid] = fmax((double)f.picket_idx[tid] - spacing / 2.0, 0.0);   // picketfence.py:1618-1627
    for (int l = tid; l < nl; l += FIN_THREADS) {
        uint32_t m = 0;
        for (int p = 0; p < np; p++) m |= (wf[l * PF_P + p].valid ? 1u : 0u) << p;
        s_vmask[l] = m;
        s_cnt[l] = __popc(m);
        if (m) atomicAdd(&s_hist[__popc(m)], 1);
        const int leaf = f.inview[l];
        s_leafnum[l] = c.p.leaf_num[leaf];
        const double lw_px = c.p.leaf_width_mm[leaf] * dpmm;
        const double lc_px = c.p.leaf_center_mm[leaf] * dpmm + n_axis_half;
        const double upper = lc_px - lw_px / 2.0 * ratio;
        const double lower = lc_px + lw_px / 2.0 * ratio;
        s_upper[l] = upper;
        s_centre[l] = (lower - upper) / 2.0 + upper;          // Line.center (core/geometry.py:556-561)
    }
    __syncthreads();
    if (wid == 0) {
        // median over the leaf rows that have at least one measurement (group_by on mlc_meas, picketfence.py:810-814): counts are
        // 1..32, lane k - 1 holds the rows with k, and its inclusive scan locates the two middle order statistics
        const int h = s_hist[lane + 1];
        int acc = h;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, acc, o);
            if (lane >= o) acc += t;
        }
        const int ng = __shfl_sync(0xffffffffu, acc, 31);
        const int total = warp_sum(h * (lane + 1));
        int status = EPID_PF_OK;
        int removed = 0;
        if (total == 0) {
            status = EPID_PF_NO_MEASUREMENTS;
        } else {
            const int ka = (ng & 1) ? ng / 2 : ng / 2 - 1, kb = ng / 2;
            const int va = __ffs(__ballot_sync(0xffffffffu, acc > ka)), vb = __ffs(__ballot_sync(0xffffffffu, acc > kb));
            const int med_twice = va + vb;                     // 2 * statistics.median
            // keep flags, and each row's offset in the table: an exclusive scan of the kept rows' counts
            int off = 0;
            for (int base = 0; base < nl; base += 32) {
                const int l = base + lane;
                const int cnt = l < nl ? s_cnt[l] : 0;
                const bool keep = cnt > 0 && 2 * cnt == med_twice;
                const int v = keep ? cnt : 0;
                int inc = v;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, inc, o);
                    if (lane >= o) inc += t;
                }
                if (l < nl) { s_keep[l] = keep ? 1 : 0; s_off[l] = off + inc - v; }
                off += __shfl_sync(0xffffffffu, inc, 31);
                removed += __popc(__ballot_sync(0xffffffffu, cnt > 0 && !keep));
            }
            if (off == 0) status = EPID_PF_EMPTY_FIT;           // a .5 median drops every row (reference: polyfit of nothing)
            else if (off > c.meas_cap) status = EPID_PF_CAPACITY;
            s_i[1] = off;
        }
        if (lane == 0) {
            s_i[0] = status;
            S.n_leaves_removed = removed;
            if (status != EPID_PF_OK) { S.status = status; f.status = status; }
        }
    }
    __syncthreads();
    if (s_i[0] != EPID_PF_OK) return;
    const int M = s_i[1];
    epid_pf_meas* meas = meas_all + (size_t)fi * c.meas_cap;
    const int npairs = nl * np;
    // ---- per-picket line fit np.polyfit(along-leaf-stack, along-travel, 1)  (picketfence.py:1881-1899): warp per picket.
    //      The second pass reloads the windows (L1 hits) instead of holding FIN_LPL slots of three doubles per lane.
    for (int p = wid; p < np; p += FIN_WARPS) {
        const double offp = s_offp[p];
        uint32_t on = 0;
        double sx = 0, sy = 0;
        int n = 0;
#pragma unroll
        for (int it = 0; it < FIN_LPL; it++) {
            const int l = it * 32 + lane;
            if (l < nl && s_keep[l] && ((s_vmask[l] >> p) & 1u)) {
                on |= 1u << it;
                const PfWin w = wf[l * PF_P + p];
                const double xv = s_upper[l];
                if (npos == 2) {
                    sx += xv * 2.0; sy += (w.l + offp) + (w.r + offp); n += 2;
                } else {
                    sx += xv; sy += fabs(w.r - w.l) / 2.0 + w.l + offp; n += 1;
                }
            }
        }
        sx = warp_sum(sx);
        sy = warp_sum(sy);
        n = warp_sum(n);
        if (n == 0) {
            if (lane == 0) { s_fit[p][0] = __longlong_as_double(0x7ff8000000000000LL); s_fit[p][1] = s_fit[p][0]; }
            continue;
        }
        const double mx_ = sx / n, my_ = sy / n;
        double sxx = 0, sxy = 0;
#pragma unroll
        for (int it = 0; it < FIN_LPL; it++) {
            if ((on >> it) & 1u) {
                const int l = it * 32 + lane;
                const PfWin w = wf[l * PF_P + p];
                const double dx = s_upper[l] - mx_;
                if (npos == 2) { sxx += 2.0 * dx * dx; sxy += dx * ((w.l + offp) - my_) + dx * ((w.r + offp) - my_); }
                else { sxx += dx * dx; sxy += dx * ((fabs(w.r - w.l) / 2.0 + w.l + offp) - my_); }
            }
        }
        sxx = warp_sum(sxx);
        sxy = warp_sum(sxy);
        if (lane == 0) {
            const double slope = sxx > 0 ? sxy / sxx : 0.0;
            s_fit[p][0] = slope;
            s_fit[p][1] = my_ - slope * mx_;
        }
    }
    __syncthreads();
    const int bad = __syncthreads_or(tid < np && s_fit[tid][0] != s_fit[tid][0]);   // a picket without measurements: polyfit([]) raises
    // ---- measurement table, leaf-major / picket-minor (= PicketFence.mlc_meas order), and its errors (picketfence.py:1701-1718):
    //      thread per (leaf, picket), plus per-thread partial aggregates.  The table is written whatever the fits.
    int m2n = 1;
    while (m2n < M * npos) m2n <<= 1;
    if (!bad)
        for (int q = M * npos + tid; q < m2n; q += FIN_THREADS) s_err[q] = __longlong_as_double(0x7ff0000000000000LL);
    int t_pass = 0, t_failed = 0, t_arg = 0x7fffffff, t_loc = 0;
    double t_max = -1.0;
#pragma unroll 1
    for (int t = tid; t < npairs; t += FIN_THREADS) {
        const int l = t / np, p = t - l * np;
        const uint32_t vm = s_vmask[l];
        if (!s_keep[l] || !((vm >> p) & 1u)) continue;
        const int q = s_off[l] + __popc(vm & ((1u << p) - 1u));
        const PfWin w = wf[l * PF_P + p];
        epid_pf_meas& m = meas[q];
        m.leaf_num = s_leafnum[l];
        m.picket = p;
        const double offp = s_offp[p];
        double pos0, pos1;
        if (npos == 2) {
            pos0 = w.l + offp;
            pos1 = w.r + offp;
        } else {
            pos0 = fabs(w.r - w.l) / 2.0 + w.l + offp;                       // center_idx (core/profile.py:322-327)
            pos1 = 0.0;
        }
        m.position[0] = pos0;
        m.position[1] = pos1;
        m.width_mm = (fmax(w.r, w.l) - fmin(w.r, w.l)) / dpmm;                // field_width_px / dpmm
        if (bad) continue;
        const double fitv = s_fit[p][0] * s_centre[l] + s_fit[p][1];
        const double tol = c.p.tolerance;
        double e0, e1 = 0.0;
        int ok1 = 1;
        if (npos == 2) {
            const double half_gap = c.p.nominal_gap_mm / 2.0 * dpmm;     // the marker lines of the two banks: fit -+ half the gap
            e0 = (pos0 - (fitv - half_gap)) / dpmm;
            e1 = (pos1 - (fitv + half_gap)) / dpmm;
            ok1 = fabs(e1) < tol ? 1 : 0;
            s_err[2 * q] = fabs(e0);
            s_err[2 * q + 1] = fabs(e1);
        } else {
            e0 = (pos0 - fitv) / dpmm;
            s_err[q] = fabs(e0);
        }
        const int ok0 = fabs(e0) < tol ? 1 : 0;
        m.error[0] = e0;
        m.error[1] = e1;
        m.passed[0] = ok0;
        m.passed[1] = ok1;
        t_pass += ok0 + (npos == 2 ? ok1 : 0);
        if (!(ok0 && ok1)) t_failed++;
        const double me = fmax(fmax(0.0, fabs(e0)), fabs(e1));
        if (me > t_max) {              // q grows with t: first maximum of this thread's subsequence, with its picket, row and bank
            t_max = me;
            t_arg = q;
            t_loc = (npos == 2 && !(fabs(e0) > fabs(e1)) ? 1 : 0) | (p << 1) | (l << 6);
        }
    }
    if (bad) {
        if (tid == 0) { S.status = EPID_PF_EMPTY_FIT; f.status = EPID_PF_EMPTY_FIT; }
        return;
    }
    // block reduction; first maximum in table order = stable descending sort .first()
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double om = __shfl_xor_sync(0xffffffffu, t_max, o);
        const int oa = __shfl_xor_sync(0xffffffffu, t_arg, o), ol = __shfl_xor_sync(0xffffffffu, t_loc, o);
        if (om > t_max || (om == t_max && oa < t_arg)) { t_max = om; t_arg = oa; t_loc = ol; }
    }
    t_pass = warp_sum(t_pass);
    t_failed = warp_sum(t_failed);
    if (lane == 0) { s_rmax[wid] = t_max; s_rarg[wid] = t_arg; s_rloc[wid] = t_loc; s_rpass[wid] = t_pass; s_rfail[wid] = t_failed; }
    __syncthreads();
    // ---- aggregates: warp 0, lane per picket
    if (wid == 0) {
        double max_err = lane < FIN_WARPS ? s_rmax[lane] : -2.0;
        int arg = lane < FIN_WARPS ? s_rarg[lane] : 0x7fffffff, loc = lane < FIN_WARPS ? s_rloc[lane] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double om = __shfl_xor_sync(0xffffffffu, max_err, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o), ol = __shfl_xor_sync(0xffffffffu, loc, o);
            if (om > max_err || (om == max_err && oa < arg)) { max_err = om; arg = oa; loc = ol; }
        }
        const int n_pass = warp_sum(lane < FIN_WARPS ? s_rpass[lane] : 0);
        const int n_failed = warp_sum(lane < FIN_WARPS ? s_rfail[lane] : 0);
        const double cax = s_cax, xmid = s_xmid;
        double d2c = 0.0, deg = 0.0;
        if (lane < np) {
            const double slope = s_fit[lane][0], icpt = s_fit[lane][1];
            S.fit_slope[lane] = slope;
            S.fit_intercept[lane] = icpt;
            d2c = (cax - (slope * xmid + icpt)) / dpmm;
            S.offsets_from_cax_mm[lane] = d2c;
            deg = slope * (180.0 / 3.14159265358979323846);
        }
        // stable rank of the offset (a NaN offset, from a NaN cax override, ranks after the numbers), and the sums in picket order
        const bool nan_me = d2c != d2c;
        int rank = 0;
        double skew = 0.0;
        for (int p = 0; p < np; p++) {
            const double o = __shfl_sync(0xffffffffu, d2c, p);
            skew += __shfl_sync(0xffffffffu, deg, p);
            const bool nan_o = o != o;
            rank += (nan_me ? (!nan_o || p < lane) : (!nan_o && (o < d2c || (o == d2c && p < lane)))) ? 1 : 0;
        }
        if (lane < np) s_srt[rank] = d2c;
        __syncwarp();
        const double gap = lane + 1 < np ? fabs(s_srt[lane] - s_srt[lane + 1]) : 0.0;
        double sp = 0.0;
        for (int p = 0; p + 1 < np; p++) sp += __shfl_sync(0xffffffffu, gap, p);
        if (lane == 0) {
            const int n_tot = s_i[1] * npos;
            S.n_meas = s_i[1];
            S.percent_passing = 100.0 * (double)n_pass / (double)n_tot;
            S.max_error_mm = max_err;
            S.max_error_picket = (loc >> 1) & (PF_P - 1);
            S.max_error_leaf = s_leafnum[loc >> 6];
            S.max_error_bank = loc & 1;
            S.passed = n_pass == n_tot ? 1 : 0;
            S.n_failed = n_failed;
            S.cax_px = cax;
            S.mlc_skew = skew / (double)np;
            S.mean_picket_spacing_mm = np > 1 ? sp / (double)(np - 1) : __longlong_as_double(0x7ff8000000000000LL);
        }
    }
    // ---- picket widths (picketfence.py:471-491): warp per picket, rank sort of <= 160 widths in shared memory
    for (int p = wid; p < np; p += FIN_WARPS) {
        double* wb = s_wbuf[wid];
        double* ws = s_wsort[wid];
        int n = 0;
#pragma unroll
        for (int it = 0; it < FIN_LPL; it++) {
            const int l = it * 32 + lane;
            const bool on = l < nl && s_keep[l] && ((s_vmask[l] >> p) & 1u);
            const unsigned b = __ballot_sync(0xffffffffu, on);
            if (on) {
                const PfWin w = wf[l * PF_P + p];
                wb[n + __popc(b & ((1u << lane) - 1u))] = (fmax(w.r, w.l) - fmin(w.r, w.l)) / dpmm;
            }
            n += __popc(b);
        }
        __syncwarp();
        for (int e = lane; e < n; e += 32) {
            const double v = wb[e];
            int rank = 0;
            for (int j = 0; j < n; j++) {
                const double o = wb[j];
                rank += (o < v || (o == v && j < e)) ? 1 : 0;
            }
            ws[rank] = v;
        }
        __syncwarp();
        if (lane == 0) {
            double sum = 0.0;
            for (int j = 0; j < n; j++) sum += wb[j];      // table order, like the reference's list
            S.picket_width_max[p] = ws[n - 1];
            S.picket_width_min[p] = ws[0];
            S.picket_width_mean[p] = sum / (double)n;
            S.picket_width_median[p] = (n & 1) ? ws[n / 2] : (ws[n / 2 - 1] + ws[n / 2]) / 2.0;
        }
        __syncwarp();
    }
    // ---- median of |errors| (np.median)
    __syncthreads();
    {
        const int ne = M * npos;
        const double med = block_median_nonneg_f64(s_err, ne);
        if (tid == 0) S.abs_median_error_mm = med;
    }
}

int launch_pf_finalize(epid_ctx* ctx, cudaStream_t stream, const PfConst* cst, PfFrame* fr, const PfWin* wins, epid_pf_summary* summ,
                       epid_pf_meas* meas, int n, int meas_cap) {
    int m2 = 1;
    while (m2 < 2 * meas_cap) m2 <<= 1;
    const size_t smem = sizeof(double) * m2;
    if (smem > 16 * 1024) EPID_SMEM_OPT_IN(ctx, k_pf_finalize, smem);
    k_pf_finalize<<<n, FIN_THREADS, smem, stream>>>(cst, fr, wins, summ, meas);
    ctx->launches++;
    EPID_CUDA(cudaGetLastError());
    return EPID_OK;
}

}  // namespace epid
