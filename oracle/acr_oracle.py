"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

pylinac.ct's Slice branch of get_regions (ct.py:3326-3340: Otsu over skimage.draw.disk(image centre, 110 mm) of the smoothed edges of
the unclipped HU, times 0.8) for Slice.phantom_roi (ct.py:381-433) and for get_regions(slice) with its defaults, the region table
CatPhanBase.find_phantom_roll (ct.py:2522-2563) reads.  Built on oracle/skimage_ct.py and oracle/ct_oracle.py, which it extends
without changing them:

    draw.disk(center, radius, shape)   oracle/skimage_draw.py's rule with skimage's clipping of the bounding box to `shape`
    measure.regionprops                label, coords, area, bbox / bbox_area (area_bbox), centroid, area_filled / filled_area
                                       (ndimage.binary_fill_holes of the region's bbox crop) and eccentricity (skimage's raw and
                                       central moments by np.dot over the crop, the inertia tensor and np.linalg.eigvalsh)

Restated without the skimage source at hand (UNPINNED, like the other skimage restatements, DESIGN.md sections 1.1 and 8.5).
"""
from __future__ import annotations

import types

import numpy as np
from scipy import ndimage

from oracle import ct_oracle, skimage_ct, skimage_shim

OK, NO_EDGES, NO_REGIONS, WRONG_SIZE = ct_oracle.OK, ct_oracle.NO_EDGES, ct_oracle.NO_REGIONS, ct_oracle.WRONG_SIZE


def disk(center, radius, shape=None):
    """skimage.draw.disk(center, radius, shape): the bounding box ceil(centre - radius) .. floor(centre + radius), clipped to `shape`,
    the float offsets from the centre measured from the clipped box's corner, ``(r / radius)**2 + (c / radius)**2 < 1``, raster
    order"""
    center = np.array(center, dtype=float)
    upper_left = np.ceil(center - radius).astype(int)
    lower_right = np.floor(center + radius).astype(int)
    if shape is not None:
        upper_left = np.maximum(upper_left, np.array([0, 0]))
        lower_right = np.minimum(lower_right, np.array(shape[:2]) - 1)
    shifted = center - upper_left
    bounding = lower_right - upper_left + 1
    r_lim, c_lim = np.ogrid[0:float(bounding[0]), 0:float(bounding[1])]
    r, c = r_lim - shifted[0], c_lim - shifted[1]
    rr, cc = np.nonzero((r / radius) ** 2 + (c / radius) ** 2 < 1)
    return rr + upper_left[0], cc + upper_left[1]


def _moments_central(image, center, order=3):
    calc = image.astype(np.float64)
    for dim, dim_length in enumerate(image.shape):
        delta = np.arange(dim_length, dtype=np.float64) - center[dim]
        powers_of_delta = delta[:, np.newaxis] ** np.arange(order + 1, dtype=np.float64)
        calc = np.rollaxis(calc, dim, image.ndim)
        calc = np.dot(calc, powers_of_delta)
        calc = np.rollaxis(calc, -1, dim)
    return calc


class Region:
    def __init__(self, lab, coords, crop):
        self.label = lab
        self.coords = coords
        self.area = len(coords)
        self.image = crop
        lo = coords.min(axis=0)
        hi = coords.max(axis=0) + 1
        self.bbox = (int(lo[0]), int(lo[1]), int(hi[0]), int(hi[1]))
        self.bbox_area = self.area_bbox = int(crop.size)
        self.filled_area = self.area_filled = int(np.sum(ndimage.binary_fill_holes(crop)))

    @property
    def centroid(self):
        return tuple(self.coords.mean(axis=0))

    @property
    def inertia_tensor(self):
        img = self.image.astype(np.uint8)
        m = _moments_central(img, (0, 0))
        local = (m[1, 0] / m[0, 0], m[0, 1] / m[0, 0])
        mu = _moments_central(img, local)
        mu0 = mu[0, 0]
        t = np.zeros((2, 2))
        t[0, 0] = mu[0, 2] / mu0
        t[1, 1] = mu[2, 0] / mu0
        t[0, 1] = t[1, 0] = -mu[1, 1] / mu0
        return t

    @property
    def eccentricity(self):
        ev = np.clip(np.linalg.eigvalsh(self.inertia_tensor), 0, None)
        l1, l2 = sorted(ev, reverse=True)
        if l1 == 0:
            return 0
        return float(np.sqrt(1 - l2 / l1))


def regionprops(label_image, intensity_image=None, **kwargs):
    label_image = np.asarray(label_image)
    out = []
    for lab in range(1, int(label_image.max()) + 1):
        coords = np.argwhere(label_image == lab)
        lo, hi = coords.min(axis=0), coords.max(axis=0) + 1
        out.append(Region(lab, coords, label_image[lo[0]:hi[0], lo[1]:hi[1]] == lab))
    return out


def disk_threshold(smoothed, radius):
    """threshold_otsu of the smoothed edges inside skimage.draw.disk(image centre, radius), times 0.8"""
    h, w = smoothed.shape
    rr, cc = disk((h / 2 - 0.5, w / 2 - 0.5), radius, shape=smoothed.shape)
    return skimage_ct.threshold_otsu(smoothed[rr, cc]) * 0.8


def _slice_stages(raw, slope, intercept, radius):
    hu = np.asarray(raw).astype(np.float64) * float(slope) + float(intercept)
    edges = skimage_ct.scharr(hu)
    smoothed = skimage_ct.gaussian(edges, sigma=1)
    return hu, edges, smoothed, disk_threshold(smoothed, radius)


def localize_slice(raw, slope, intercept, catphan_size, clear_borders, radius):
    """Slice.phantom_roi on the Slice branch: ct_oracle.localize_slice's dict, with the unclipped edges as "scharr" """
    hu, edges, smoothed, thres = _slice_stages(raw, slope, intercept, radius)
    out = {"hu": hu, "max_edge": float(np.max(edges)), "n_regions": 0, "label": -1, "area": 0, "centroid_row": np.nan,
           "centroid_col": np.nan}
    if out["max_edge"] < 0.1:
        out["status"] = NO_EDGES
        return out
    bw = smoothed > thres
    if clear_borders:
        bw = skimage_shim.clear_border(bw, buffer_size=min(int(max(bw.shape) / 100), 3))
    bw = ndimage.binary_fill_holes(bw)
    labels, num = skimage_ct.label(bw, return_num=True)
    regions = regionprops(labels)
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


def slice_regions(raw, slope, intercept, radius):
    """get_regions(slice) with its defaults -> (regions in label order, threshold, max_edge, labels)"""
    hu, edges, smoothed, thres = _slice_stages(raw, slope, intercept, radius)
    bw = smoothed > thres
    bw = skimage_shim.clear_border(bw, buffer_size=min(int(max(bw.shape) / 100), 3))
    labels = skimage_ct.label(bw)
    return regionprops(labels), float(thres), float(np.max(edges)), labels


def region_rows(regions, width):
    """the epid_ct_region fields of each region: label, first, area, filled_area, bbox, sum_r, sum_c and the moments about the bbox
    corner (exact integers)"""
    rows = []
    for r in regions:
        c = r.coords.astype(np.int64)
        dy, dx = c[:, 0] - r.bbox[0], c[:, 1] - r.bbox[1]
        rows.append(dict(label=r.label, first=int(c[0, 0] * width + c[0, 1]), area=r.area, filled_area=r.filled_area, bbox=r.bbox,
                         sum_r=int(c[:, 0].sum()), sum_c=int(c[:, 1].sum()), m_rr=int((dy * dy).sum()), m_cc=int((dx * dx).sum()),
                         m_rc=int((dy * dx).sum())))
    return rows


def install():
    """bind the restatements into the stub-imported pylinac.ct (over oracle/skimage_ct.py's); returns that module"""
    ct = skimage_ct.install()
    ct.draw = types.SimpleNamespace(disk=disk)
    ct.measure = types.SimpleNamespace(label=skimage_ct.label, regionprops=regionprops)
    return ct
