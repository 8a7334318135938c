"""The moments-based MTF of Hander et al. 1997 (core/mtf.py:194-260): host scalar math on the mean and standard deviation of
high-contrast bar-pattern ROIs, in the reference's own expressions (``math.sqrt``, ``np.log``), so it raises where the reference
raises: ``ValueError`` (math domain error) where ``std**2 < mean`` and ``ZeroDivisionError`` on a blank ROI.  The ROI statistics come
from the device (core/roi.py)."""
from __future__ import annotations

import math
from collections.abc import Sequence

import numpy as np

from .roi import HighContrastDiskROI


def moments_mtf(mean: float, std: float) -> float:
    """The moments-based MTF based on Hander et al 1997 Equation 8."""
    return math.sqrt(2 * (std**2 - mean)) / mean


def moments_fwhm(width: float, mean: float, std: float) -> float:
    """The moments-based FWHM based on Hander et al 1997 Equation A8; `width` is the bar width in mm."""
    return 1.058 * width * math.sqrt(np.log(mean / (math.sqrt(2 * (std**2 - mean)))))


class MomentMTF:
    """A moments-based MTF of ROIs with the given line pairs per mm, means and standard deviations, paired in order."""

    mtfs: dict[float, float]
    fwhms: dict[float, float]

    def __init__(self, lpmms: Sequence[float], means: Sequence[float], stds: Sequence[float]):
        self.mtfs = {}
        self.fwhms = {}
        for lpmm, mean, std in zip(lpmms, means, stds):
            bar_width = 1 / (2 * lpmm)  # lp is 2 bars
            self.mtfs[lpmm] = moments_mtf(mean, std)
            self.fwhms[lpmm] = moments_fwhm(bar_width, mean, std)

    @classmethod
    def from_high_contrast_diskset(cls, lpmms: Sequence[float], diskset: Sequence[HighContrastDiskROI]) -> MomentMTF:
        """Construct the MTF using high contrast disks from the ROI module."""
        means = [roi.mean for roi in diskset]
        stds = [roi.std for roi in diskset]
        return cls(lpmms, means, stds)
