"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

scikit-image is not installed in this container.  The reference's ``gamma_2d`` (core/gamma.py:229-330) takes its search offsets
from ``skimage.draw.disk``; this module restates that one function so that the UNMODIFIED reference can run (the golden generator
rebinds ``pylinac.core.gamma.disk`` to it) and so that the oracle and the tests use the same offsets.
"""
from __future__ import annotations

import numpy as np


def disk(center, radius, shape=None):
    """skimage.draw.disk(center, radius) = ellipse(r, c, radius, radius) with rotation 0: the bounding box ceil(centre - radius) ..
    floor(centre + radius), float ogrid offsets from the centre, membership ``(r / radius)**2 + (c / radius)**2 < 1`` (the rotation
    terms multiply by cos 0 = 1 and sin 0 = 0 exactly), np.nonzero (raster) order.  The floating-point test is not the integer
    r**2 + c**2 < radius**2: at radius 41 it keeps (+-40, +-9) and (+-9, +-40), which lie on the circle.  Restated without the
    skimage source at hand (UNPINNED); ``shape`` clipping is not used by the reference's gamma_2d and not restated."""
    if shape is not None:
        raise NotImplementedError("disk(shape=...) is not restated")
    center = np.array(center, dtype=float)
    upper_left = np.ceil(center - radius).astype(int)
    lower_right = np.floor(center + radius).astype(int)
    shifted = center - upper_left
    bounding = lower_right - upper_left + 1
    r_lim, c_lim = np.ogrid[0:float(bounding[0]), 0:float(bounding[1])]
    r, c = r_lim - shifted[0], c_lim - shifted[1]
    rr, cc = np.nonzero((r / radius) ** 2 + (c / radius) ** 2 < 1)
    return rr + upper_left[0], cc + upper_left[1]
