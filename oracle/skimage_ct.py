"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

The skimage calls of pylinac.ct's localization (ct.py:381-433 Slice.phantom_roi, ct.py:3315-3348 get_regions), restated on numpy /
scipy and installed into the stub-imported ``pylinac.ct`` by :func:`install`:

    filters.scharr          per axis ndimage.convolve with the [1, 0, -1] x [3, 10, 3] / 16 kernel (mode 'reflect'), then
                            sqrt(a0 * a0 + a1 * a1) / sqrt(2)
    filters.gaussian        ndimage.gaussian_filter(mode='nearest', truncate=4) of a float64 image
    filters.threshold_otsu  np.histogram(image, 256) centres, the between-class variance argmax; a constant image returns its value
    segmentation.clear_border(buffer_size)   oracle/skimage_shim.py's
    measure.label           full (8-) connectivity, raster-order numbering
    measure.regionprops     area, filled_area (asserted equal to area: after binary_fill_holes no background is enclosed) and
                            centroid = coords.mean(axis=0)

Restated without the skimage source at hand (UNPINNED, like the other skimage restatements, DESIGN.md sections 1.1 and 8.5).
binary_fill_holes and gaussian_filter are the real scipy.
"""
from __future__ import annotations

import types

import numpy as np
from scipy import ndimage

from oracle import skimage_shim

_SMOOTH = np.array([3, 10, 3]) / 16.0


def scharr(image):
    image = np.asarray(image, dtype=np.float64)
    output = np.zeros(image.shape)
    for edge_dim in range(2):
        kernel = np.array([1, 0, -1]).reshape((3, 1) if edge_dim == 0 else (1, 3))
        kernel = kernel * _SMOOTH.reshape((1, 3) if edge_dim == 0 else (3, 1))
        ax = ndimage.convolve(image, kernel, mode="reflect")
        ax *= ax
        output += ax
    return np.sqrt(output) / np.sqrt(2)


def gaussian(image, sigma=1, **kwargs):
    return ndimage.gaussian_filter(np.asarray(image, dtype=np.float64), sigma, mode="nearest", truncate=4.0)


def threshold_otsu(image, nbins=256):
    image = np.asarray(image)
    first = image.reshape(-1)[0]
    if np.all(image == first):
        return first
    counts, edges = np.histogram(image.reshape(-1), bins=nbins)
    centers = (edges[:-1] + edges[1:]) / 2.0
    weight1 = np.cumsum(counts)
    weight2 = np.cumsum(counts[::-1])[::-1]
    mean1 = np.cumsum(counts * centers) / weight1
    mean2 = (np.cumsum((counts * centers)[::-1]) / weight2[::-1])[::-1]
    variance12 = weight1[:-1] * weight2[1:] * (mean1[:-1] - mean2[1:]) ** 2
    return centers[np.argmax(variance12)]


def label(image, return_num=False, connectivity=None, **kwargs):
    lab = skimage_shim.label(image, connectivity=connectivity)
    return (lab, int(lab.max())) if return_num else lab


class _Region:
    def __init__(self, lab, coords):
        self.label = lab
        self.coords = coords
        self.area = len(coords)

    @property
    def filled_area(self):
        return self.area

    @property
    def centroid(self):
        return tuple(self.coords.mean(axis=0))


def regionprops(label_image, intensity_image=None, **kwargs):
    label_image = np.asarray(label_image)
    out = []
    for lab in range(1, int(label_image.max()) + 1):
        coords = np.argwhere(label_image == lab)
        region = label_image == lab
        lo, hi = coords.min(axis=0), coords.max(axis=0) + 1
        crop = region[lo[0]:hi[0], lo[1]:hi[1]]
        assert ndimage.binary_fill_holes(crop).sum() == len(coords), "filled_area differs from area"
        out.append(_Region(lab, coords))
    return out


def install():
    """bind the restatements into the stub-imported pylinac.ct; returns that module"""
    from pylinac import ct

    ct.filters = types.SimpleNamespace(scharr=scharr, gaussian=gaussian, threshold_otsu=threshold_otsu)
    ct.segmentation = types.SimpleNamespace(clear_border=skimage_shim.clear_border)
    ct.measure = types.SimpleNamespace(label=label, regionprops=regionprops)
    ct.ndimage = ndimage
    return ct
