"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

pylinac.ct's per-slice localization (Slice.phantom_roi, ct.py:381-433, with get_regions' ndarray branch, ct.py:3315-3348) in numpy,
stage by stage, so that the device's epid_ct_localize can be compared with it plane by plane.  The skimage calls are
oracle/skimage_ct.py's restatements; binary_fill_holes is scipy's.
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage

from oracle import skimage_ct

OK, NO_EDGES, NO_REGIONS, WRONG_SIZE = 0, 1, 2, 3


def localize_slice(raw, slope, intercept, catphan_size, clear_borders):
    """-> dict of the stages (hu, max_edge, scharr of the clipped slice, smoothed, threshold, filled mask, labels) and the row
    (status, n_regions, label, area, centroid_row, centroid_col); stages after a failed edge check are absent."""
    hu = np.asarray(raw).astype(np.float64) * float(slope) + float(intercept)
    out = {"hu": hu, "max_edge": float(np.max(skimage_ct.scharr(hu))), "n_regions": 0, "label": -1, "area": 0,
           "centroid_row": np.nan, "centroid_col": np.nan}
    if out["max_edge"] < 0.1:
        out["status"] = NO_EDGES
        return out
    clipped = np.clip(hu, a_min=-1000, a_max=1000)
    edges = skimage_ct.scharr(clipped)
    smoothed = skimage_ct.gaussian(edges, sigma=1)
    thres = skimage_ct.threshold_otsu(smoothed)
    bw = smoothed > thres
    if clear_borders:
        bw = skimage_ct.skimage_shim.clear_border(bw, buffer_size=min(int(max(bw.shape) / 100), 3))
    bw = ndimage.binary_fill_holes(bw)
    labels, num = skimage_ct.label(bw, return_num=True)
    regions = skimage_ct.regionprops(labels)
    out.update(scharr=edges, smoothed=smoothed, threshold=float(thres), filled=bw, labels=labels, n_regions=num)
    if num < 1:
        out["status"] = NO_REGIONS
        return out
    region = sorted(regions, key=lambda x: np.abs(x.filled_area - catphan_size))[0]
    cy, cx = region.centroid
    first = region.coords[0]
    out.update(label=int(first[0] * hu.shape[1] + first[1]), area=region.area, centroid_row=float(cy), centroid_col=float(cx))
    too_large = catphan_size * 1.3 < region.filled_area
    too_small = region.filled_area < catphan_size / 1.3
    out["status"] = WRONG_SIZE if (too_large or too_small) else OK
    return out
