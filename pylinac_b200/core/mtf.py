"""The relative MTF of disk maxima and minima (core/mtf.py:32-115) and the moments-based MTF of Hander et al. 1997
(core/mtf.py:194-260): host scalar math on the statistics of high-contrast ROIs, in the reference's own expressions, so they warn and
raise where the reference does (the moments MTF: ``ValueError`` (math domain error) where ``std**2 < mean`` and ``ZeroDivisionError``
on a blank ROI).  The ROI statistics come from the device (core/roi.py)."""
from __future__ import annotations

import math
import warnings
from collections.abc import Sequence

import numpy as np

from .contrast import michelson
from .roi import HighContrastDiskROI, RectangleROI


def _interp1d_extrapolate(x, y, x_new: float) -> np.ndarray:
    """scipy.interpolate.interp1d(x, y, fill_value="extrapolate")(x_new) for 1-D x, y and a scalar x_new: x sorted by a stable
    argsort, the interval by searchsorted clipped to [1, len - 1], and the two-term linear expression of interp1d._call_linear."""
    x = np.array(x, dtype=np.float64)
    y = np.array(y, dtype=np.float64)
    ind = np.argsort(x, kind="mergesort")
    x, y = x[ind], y[ind]
    x_new = np.asarray(x_new, dtype=np.float64).ravel()
    idx = np.searchsorted(x, x_new).clip(1, len(x) - 1).astype(int)
    lo, hi = idx - 1, idx
    x_lo, x_hi, y_lo, y_hi = x[lo], x[hi], y[lo], y[hi]
    y_new = ((x_new - x_lo) / (x_hi - x_lo)) * y_hi + ((x_hi - x_new) / (x_hi - x_lo)) * y_lo
    return y_new.reshape(())


class MTF:
    """The relative MTF: the Michelson contrast of each line-pair region's maximum and minimum, normalized to the first spacing."""

    def __init__(self, lp_spacings: Sequence[float], lp_maximums: Sequence[float], lp_minimums: Sequence[float]):
        """lp_spacings: line pairs per unit distance; lp_maximums / lp_minimums: the maximum / minimum of each region."""
        self.spacings = lp_spacings
        self.maximums = lp_maximums
        self.minimums = lp_minimums
        if len(lp_spacings) != len(lp_maximums) != len(lp_minimums):
            raise ValueError("The number of MTF spacings, maximums, and minimums must be equal.")
        if len(lp_spacings) < 2 or len(lp_maximums) < 2 or len(lp_minimums) < 2:
            raise ValueError("The number of MTF spacings, maximums, and minimums must be greater than 1.")
        self.mtfs = {}
        self.norm_mtfs = {}
        for spacing, max, min in zip(lp_spacings, lp_maximums, lp_minimums):
            arr = np.array((max, min))
            self.mtfs[spacing] = michelson(arr)
        # sort according to spacings
        self.mtfs = {k: v for k, v in sorted(self.mtfs.items(), key=lambda x: x[0])}
        for key, value in self.mtfs.items():
            self.norm_mtfs[key] = value / self.mtfs[lp_spacings[0]]  # normalize to first region
        # the MTF should drop monotonically: a positive delta between consecutive MTFs means it rose
        max_delta = np.max(np.diff(list(self.norm_mtfs.values())))
        if max_delta > 0:
            warnings.warn("The MTF does not drop monotonically; be sure the ROIs are correctly aligned.")

    def relative_resolution(self, x: float = 50) -> float:
        """The line pair value at the given rMTF percentage `x` (0 to 100), extrapolated linearly beyond the measured range."""
        if not 0 <= x <= 100:
            raise ValueError(f"Argument 'x' needs to be between 0 and 100; got {x}")
        mtf = _interp1d_extrapolate(list(self.norm_mtfs.values()), list(self.norm_mtfs.keys()), x / 100)
        if mtf > max(self.spacings):
            warnings.warn(f"MTF resolution wasn't calculated for {x}% that was asked for. The value returned is an extrapolation. "
                          f"Use a higher % MTF to get a non-interpolated value.")
        return float(mtf)

    @classmethod
    def from_high_contrast_diskset(cls, spacings: Sequence[float], diskset: Sequence[HighContrastDiskROI | RectangleROI]) -> MTF:
        """Construct the MTF using high contrast disks from the ROI module."""
        maximums = [roi.max for roi in diskset]
        minimums = [roi.min for roi in diskset]
        return cls(spacings, maximums, minimums)


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
