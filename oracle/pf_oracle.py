"""ORACLE (test infrastructure; never imported by the product path).

CPU restatement of ``PicketFence(image).analyze()`` + ``results_data()`` of the
reference as one pure function ``frame -> dict`` built on numpy + scipy (the
third-party routines the reference itself calls: scipy 1.18.1 / numpy 2.3.5 in
this image; the reference pins ranges only, pyproject.toml:29-46).

Pinned against the unmodified reference (stub-imported, oracle/refstub.py) by
``tests/golden/make_pf_golden.py`` -> ``tests/golden/pf_*.npz`` and by
``tests/test_oracle_pf.py``.

Every step cites the reference line it follows (``pf:`` = pylinac/picketfence.py,
``img:`` = pylinac/core/image.py, ``au:`` = pylinac/core/array_utils.py,
``prof:`` = pylinac/core/profile.py).
"""
from __future__ import annotations

import statistics

import numpy as np
from scipy import ndimage, signal
from scipy.interpolate import UnivariateSpline

UP_DOWN = 0
LEFT_RIGHT = 1

# pf:103-135 -- (count, width mm) runs
MLC_ARRANGEMENTS = {
    "Millennium": [(10, 10), (40, 5), (10, 10)],
    "HD Millennium": [(14, 5), (32, 2.5), (14, 5)],
    "B Mod": [(40, 4)],
    "Agility": [(80, 5)],
    "MLCi": [(40, 10)],
    "Halcyon distal": [(28, 10)],
    "Halcyon proximal": [(29, 10)],
}


def mlc_arrangement(runs, offset=0.0):
    """pf:71-100: leaf centres (mm, mean-subtracted), widths, leaf numbers (descending)."""
    centers, widths = [], []
    rolling_edge = 0
    for leaf_num, width in runs:
        centers += np.arange(start=rolling_edge + width / 2, stop=leaf_num * width + rolling_edge + width / 2, step=width).tolist()
        rolling_edge = centers[-1] + width / 2
        widths += [width] * leaf_num
    mean = np.mean(centers)
    centers = [c - mean + offset for c in centers]
    leaves = np.arange(1, len(centers) + 1, dtype=int)[::-1].tolist()
    return leaves, centers, widths


def _invert(a):
    return -a + a.max() + a.min()  # au:75-77 (dtype preserving, modular for uint)


def has_noise(a) -> bool:
    """pf:229-238"""
    mn, mx = a.min(), a.max()
    near_min, near_max = np.percentile(a, [0.5, 99.5])
    max_is_extreme = mx > near_max * 1.25
    min_is_extreme = (mn < near_min * 0.75) and (abs(mn - near_min) > 0.1 * (near_max - near_min))
    return bool(max_is_extreme or min_is_extreme)


def orientation_ranges(img):
    """pf:1501-1526 on the ground + normalised image: (orientation, row range, column range).  The orientation is LEFT_RIGHT
    when the p99 - p85 range of the per-column sums is below that of the per-row sums."""
    temp = img.copy()
    med = np.median(temp)
    temp[temp < med] = med
    row_sum = np.sum(temp, 0)
    col_sum = np.sum(temp, 1)
    row80, row90 = np.percentile(row_sum, [85, 99])
    col80, col90 = np.percentile(col_sum, [85, 99])
    row_range, col_range = row90 - row80, col90 - col80
    return (LEFT_RIGHT if row_range < col_range else UP_DOWN), row_range, col_range


def corner_inversion_needed(a, box_size=10, position=(0.01, 0.01)) -> bool:
    """img:881-897"""
    row_pos = max(int(position[0] * a.shape[0]), 1)
    col_pos = max(int(position[1] * a.shape[1]), 1)
    lt_upper = a[row_pos : row_pos + box_size, col_pos : col_pos + box_size]
    rt_upper = a[row_pos : row_pos + box_size, -col_pos - box_size : -col_pos]
    lt_lower = a[-row_pos - box_size : -row_pos, col_pos : col_pos + box_size]
    rt_lower = a[-row_pos - box_size : -row_pos, -col_pos - box_size : -col_pos]
    avg = np.mean((lt_upper, lt_lower, rt_upper, rt_lower))
    return bool(avg > np.mean(a.flatten()))


def ref_find_peaks(values, threshold=-np.inf, peak_separation=0, max_number=None, fwxm_height=0.5, min_width=0,
                   search_region=(0.0, 1.0), peak_sort="prominences", required_prominence=None):
    """prof:2545-2649 (find_peaks + _parse_peak_args)."""
    values = np.asarray(values)
    val_range = values.max() - values.min()
    if 0 <= threshold <= 1:
        threshold = values.min() + threshold * val_range
    if 0 <= peak_separation <= 1:
        peak_separation = max(int(peak_separation * len(values)), 1)
    if max(search_region) <= 1:
        shift = int(search_region[0] * len(values))
        trimmed = values[int(search_region[0] * len(values)) : int(search_region[1] * len(values))]
    else:
        trimmed = values[search_region[0] : search_region[1]]
        shift = search_region[0]
    idxs, props = signal.find_peaks(trimmed, rel_height=(1 - fwxm_height), width=min_width, height=threshold,
                                    distance=peak_separation, prominence=required_prominence)
    idxs = idxs + shift
    largest = sorted(list(np.argsort(props[peak_sort]))[::-1][:max_number])
    for k, v in props.items():
        props[k] = v[largest]
    return idxs[largest], props


def _x_at_x_idx(n, x):
    """prof:249-262 with x_values = arange(n): a k=1, s=0 spline through (i, i)."""
    f = UnivariateSpline(x=np.arange(n), y=np.arange(n), k=1, s=0)
    return float(f(x))


def fwxm_edges(values, fwxm_height=50):
    """FWXMProfile.field_edge_idx (prof:602-611) for both sides on already ground+normalised values."""
    _, props = ref_find_peaks(values, fwxm_height=fwxm_height / 100, max_number=1)
    n = len(values)
    return _x_at_x_idx(n, props["left_ips"][0]), _x_at_x_idx(n, props["right_ips"][0])


def pf_analyze(frame, dpmm, *, crop_mm=3, filter=None, mlc="Millennium", tolerance=0.5, action_tolerance=None,
               num_pickets=None, sag_adjustment=0, orientation=None, invert=False, leaf_analysis_width_ratio=0.4,
               picket_spacing=None, height_threshold=0.5, edge_threshold=1.5, peak_sort="peak_heights",
               required_prominence=0.2, fwxm=50, separate_leaves=False, nominal_gap_mm=3, sid=1000.0):
    """Returns a dict of every quantity the GPU path must reproduce.  Raises ValueError like the reference."""
    if action_tolerance is not None and tolerance < action_tolerance:
        raise ValueError("Tolerance cannot be lower than the action tolerance")  # pf:728-729
    out = {}
    a = np.asarray(frame)
    # pf:214-215  crop
    c = int(round(crop_mm * dpmm))
    if c > 0:
        a = a[c:-c, c:-c]
    if a.size == 0:
        raise ValueError("Too many pixels removed; array is empty. Pass a smaller crop value.")
    # pf:221-227  noise loop
    n_med = 0
    safety = 5
    while has_noise(a) and safety > 0:
        a = ndimage.median_filter(a, size=3)
        safety -= 1
        n_med += 1
    out["noise_median_passes"] = n_med
    # pf:219  corner inversion
    inv = corner_inversion_needed(a)
    out["corner_inverted"] = inv
    if inv:
        a = _invert(a)
    # pf:320-323
    if isinstance(filter, int):
        a = ndimage.median_filter(a, size=filter)
    a = a - a.min()  # ground (au:102, value=0 keeps dtype)
    img = a / a.max()  # normalize -> float64 (au:64-71)
    if invert:  # pf:738-739
        img = _invert(img)
    H, W = img.shape
    out["shape"] = (H, W)

    def _orientation():
        return orientation_ranges(img)[0]

    if orientation is None:
        orient = None
    else:
        orient = UP_DOWN if str(orientation).lower().startswith("u") or orientation == UP_DOWN else LEFT_RIGHT
    # pf:743-745 sag adjustment (forces the orientation property to evaluate first)
    if sag_adjustment != 0:
        sag_px = int(round(sag_adjustment * dpmm))
        if orient is None:
            orient = _orientation()
        img = np.roll(img, sag_px, axis=0 if orient == UP_DOWN else 1)
    if orient is None:
        orient = _orientation()
    out["orientation"] = orient

    # pf:747-759 picket search
    leaf_prof = np.mean(img, 0) if orient == UP_DOWN else np.mean(img, 1)
    leaf_prof = leaf_prof / leaf_prof.max()  # MultiProfile.normalize (prof:107-109 -> au.normalize)
    out["leaf_profile"] = leaf_prof
    _, props = ref_find_peaks(leaf_prof, threshold=height_threshold, peak_separation=0.02, max_number=num_pickets,
                              peak_sort=peak_sort, required_prominence=required_prominence)
    peak_idxs = [int(round(lt + (rt - lt) / 2)) for lt, rt in zip(props["left_ips"], props["right_ips"])]  # prof:2165-2168
    peak_vals = [leaf_prof[i] for i in peak_idxs]
    if len(peak_idxs) == 0:
        raise ValueError("No pickets were found.")
    out["picket_idx"] = np.array(peak_idxs, dtype=np.int64)
    out["picket_val"] = np.array(peak_vals, dtype=np.float64)
    if picket_spacing is None:
        picket_spacing = np.median(np.diff(np.sort(peak_idxs)))  # pf:766-767
    out["picket_spacing"] = float(picket_spacing)
    spacing = picket_spacing

    runs = MLC_ARRANGEMENTS[mlc] if isinstance(mlc, str) else mlc
    leaves, centers, widths = mlc_arrangement(runs)
    n_axis = H if orient == UP_DOWN else W
    # pf:888-912
    pixel_range = n_axis / 2 - max(widths[0] * leaf_analysis_width_ratio, widths[-1] * leaf_analysis_width_ratio) * dpmm
    in_view = [(ln, cc, ww) for ln, cc, ww in zip(leaves, centers, widths) if abs(cc) < pixel_range / dpmm]

    meas = []  # dicts
    for leaf_num, center, width in in_view:
        lw_px = width * dpmm
        lc_px = center * dpmm + n_axis / 2  # pf:863-868
        for pk, (pidx, pval) in enumerate(zip(peak_idxs, peak_vals)):
            # pf:869-886
            if orient == UP_DOWN:
                left = max(int(pidx - spacing / 2), 0)
                right = min(int(pidx + spacing / 2), W)
                top = max(int(lc_px - lw_px / 2), 0)
                bottom = min(int(lc_px + lw_px / 2), H)
            else:
                top = max(int(pidx - spacing / 2), 0)
                bottom = min(int(pidx + spacing / 2), H)
                left = max(int(lc_px - lw_px / 2), 0)
                right = min(int(lc_px + lw_px / 2), W)
            win = img[top:bottom, left:right]
            # pf:847-857
            std = np.std(win, axis=1) if orient == UP_DOWN else np.std(win, axis=0)
            ok = (np.max(win) > height_threshold * pval) and (max(std) < edge_threshold * np.median(std))
            if not ok:
                continue
            # pf:1605-1628
            pix = np.median(win, axis=0) if orient == UP_DOWN else np.median(win, axis=1)
            pix = pix - pix.min()
            pix = pix / pix.max()
            # NOTE: the reference stores ``fwxm`` (pf:1563) but never forwards it to FWXMProfilePhysical
            # (pf:1610-1615), so the kiss position is always the FWHM centre.  Reproduced, not fixed.
            l_ip, r_ip = fwxm_edges(pix, 50)
            off = max(pidx - spacing / 2, 0)
            if separate_leaves:
                position = (l_ip + off, r_ip + off)
            else:
                position = (abs(r_ip - l_ip) / 2 + l_ip + off,)
            width_px = max(r_ip, l_ip) - min(r_ip, l_ip)
            meas.append(dict(leaf=leaf_num, picket=pk, lc_px=lc_px, lw_px=lw_px, position=position,
                             width_mm=width_px / dpmm))
    if not meas:
        raise ValueError("No MLC measurements were found.")
    # pf:810-824 leaf-row pruning
    by_leaf: dict = {}
    for m in meas:
        by_leaf.setdefault(m["leaf"], []).append(m)
    median_n = statistics.median([len(v) for v in by_leaf.values()])
    full = [k for k, v in by_leaf.items() if len(v) == median_n]
    # the reference keeps no count of the dropped rows: leaf rows with a measurement minus the rows kept
    out["n_leaves_removed"] = len(by_leaf) - len(full)
    meas = [m for m in meas if m["leaf"] in full]
    out["n_meas"] = len(meas)

    ratio = leaf_analysis_width_ratio
    fits = []
    for pk in range(len(peak_idxs)):
        pm = [m for m in meas if m["picket"] == pk]
        # pf:1881-1899, 1725-1743: point1 of each marker line = (position, lc - lw/2*ratio)
        xs, ys = [], []
        for m in pm:
            upper = m["lc_px"] - m["lw_px"] / 2 * ratio
            for p in m["position"]:
                xs.append(upper)  # coordinate along the leaf-stacking axis
                ys.append(p)      # coordinate along leaf travel
        fit = np.polyfit(xs, ys, 1)
        fits.append(fit)
    out["fits"] = np.array(fits)

    # pf:1701-1718 errors
    for m in meas:
        fit = np.poly1d(fits[m["picket"]])
        upper = m["lc_px"] - m["lw_px"] / 2 * ratio
        lower = m["lc_px"] + m["lw_px"] / 2 * ratio
        centre_along = (lower - upper) / 2 + upper  # Line.center (geometry.py:556-561)
        errs = []
        for p, sign in zip(m["position"], (-1, 1)):
            picket_pos = fit(centre_along)
            if separate_leaves:
                picket_pos += sign * nominal_gap_mm / 2 * dpmm
            errs.append((p - picket_pos) / dpmm)
        m["error"] = errs
        m["passed"] = [abs(e) < tolerance for e in errs]

    out["meas_leaf"] = np.array([m["leaf"] for m in meas], dtype=np.int64)
    out["meas_picket"] = np.array([m["picket"] for m in meas], dtype=np.int64)
    out["meas_position"] = np.array([m["position"] for m in meas], dtype=np.float64)
    out["meas_error"] = np.array([m["error"] for m in meas], dtype=np.float64)
    out["meas_width_mm"] = np.array([m["width_mm"] for m in meas], dtype=np.float64)

    flat_err = [e for m in meas for e in m["error"]]
    flat_pass = [p for m in meas for p in m["passed"]]
    out["percent_passing"] = float(100 * sum(1 for p in flat_pass if p) / len(flat_pass))  # pf:445-454
    out["max_error"] = float(np.max(np.abs(flat_err)))
    out["abs_median_error"] = float(np.median(np.abs(flat_err)))
    worst = sorted(meas, key=lambda m: np.max(np.abs(m["error"])), reverse=True)[0]  # pf:462-514 (stable descending)
    out["max_error_picket"] = int(worst["picket"])
    if not separate_leaves:
        out["max_error_leaf"] = int(worst["leaf"])
    else:
        out["max_error_leaf"] = ("A" if abs(worst["error"][0]) > abs(worst["error"][1]) else "B") + str(worst["leaf"])
    out["passed"] = bool(all(flat_pass))
    failing = []
    for m in meas:  # pf:519-539
        if not all(m["passed"]):
            if not separate_leaves:
                names = [m["leaf"]]
            else:
                names = [f"{pre}{m['leaf']}" for pre, ok in zip("AB", m["passed"]) if not ok]
            for nme in names:
                if nme not in failing:
                    failing.append(nme)
    out["failed_leaves"] = failing
    # pf:1905-1923 dist2cax, image.center img:526-533
    cax = ((W / 2) - 0.5) if orient == UP_DOWN else ((H / 2) - 0.5)
    length = H if orient == UP_DOWN else W
    idx = int(round(length / 2))
    d2c = []
    for fit in fits:
        y_data = np.poly1d(fit)(np.arange(length))
        d2c.append((cax - y_data[idx]) / dpmm)
    out["offsets_from_cax_mm"] = np.array(d2c)
    srt = sorted(d2c)
    out["mean_picket_spacing"] = float(np.mean([abs(srt[i] - srt[i + 1]) for i in range(len(srt) - 1)])) if len(srt) > 1 else float("nan")
    out["mlc_skew"] = float(np.mean([float(np.rad2deg(f[0])) for f in fits]))  # pf:1467-1469, 1901-1903
    out["number_of_pickets"] = len(fits)
    # pf:471-491 picket widths
    pw = np.zeros((len(fits), 4))
    for pk in range(len(fits)):
        w = [m["width_mm"] for m in meas if m["picket"] == pk]
        pw[pk] = (max(w), statistics.mean(w), statistics.median(w), min(w))
    out["picket_widths"] = pw  # columns: max, mean, median, min
    out["cax_mm"] = cax / dpmm
    return out


def primitives_plumbing(frame, sigma=2, rel_threshold=0.5):
    """BASELINE.json config 1: gaussian filter then threshold (au:133; img:797-798)."""
    g = ndimage.gaussian_filter(frame, sigma=sigma)
    t = rel_threshold * g.max()
    return np.where(g >= t, g, 0)
