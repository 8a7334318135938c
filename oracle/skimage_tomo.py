"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

``pylinac.nuclear.TomographicContrast.slice_data`` (nuclear.py:1620-1658) reads ``regionprops(...).centroid``, which the skimage
restatements of oracle/skimage_nuclear.py leave to oracle/skimage_shim.py.  The shim's centroid adds the bounding-box offset after the
mean, which rounds twice, and other goldens depend on it, so neither module changes: this one wraps the shim's regions with
skimage's centroid and :func:`install` binds it, with oracle/skimage_nuclear.py's restatements, into ``pylinac.nuclear``.
Restated without the skimage source at hand (UNPINNED, like the other skimage restatements, DESIGN.md section 8.5).
"""
from __future__ import annotations

import numpy as np

from oracle import skimage_nuclear


class _Region:
    """one region of :func:`regionprops`: the shim's region with skimage's ``centroid``"""

    def __init__(self, region, label_image):
        self._region = region
        self._label_image = label_image

    def __getattr__(self, name):
        return getattr(self._region, name)

    @property
    def centroid(self):
        """skimage's centroid: the mean of the region's global (row, col) coordinates, one rounding per axis"""
        coords = np.argwhere(self._label_image == self._region.label)
        return tuple(coords.mean(axis=0))


def regionprops(label_image, intensity_image=None, **kwargs):
    """skimage.measure.regionprops with the properties TomographicContrast.slice_data reads: ``area``, ``image`` and ``centroid``"""
    label_image = np.asarray(label_image)
    return [_Region(r, label_image) for r in skimage_nuclear.regionprops(label_image, intensity_image)]


def install():
    """oracle/skimage_nuclear.py's install(), with regionprops rebound to :func:`regionprops` (TomographicContrast reads the
    centroid)"""
    rn = skimage_nuclear.install()
    rn.regionprops = regionprops
    return rn
