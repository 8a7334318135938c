"""``DiskROI``, ``HighContrastDiskROI`` (core/roi.py:39-190, 411-478) and ``RectangleROI`` (core/roi.py:481-706): regions of an image
array and the statistics of their pixels.

A disk's pixels are ``arr[skimage.draw.disk((cy, cx), r)]`` in the reference.  Its median, mean, std, min and max come from one
device call (``epid_disk_stats``, csrc/roi.cu), equal bit for bit to numpy's over the same pixels in the same order; ``pixel_values``,
``circle_mask`` and ``masked_array`` gather on the host.  The pixel selection of a rectangle is skimage.draw.polygon's in the reference
(``pixels_flat``); here the statistics are device reductions over the same pixel set (``epid_roi_stats``, csrc/roi.cu: integer pixel
coordinates inside or on the boundary of the corner polygon the reference builds, clipped to the image).  ``pixel_array`` (non-rotated
ROIs) is a numpy view like the reference's."""
from __future__ import annotations

from collections.abc import Sequence
from functools import cached_property

import numpy as np

from .. import _native as nat
from .geometry import Circle, Point, Rectangle


def disk(center, radius, shape=None) -> tuple[np.ndarray, np.ndarray]:
    """skimage.draw.disk(center, radius, shape): (rr, cc) of the pixels whose offsets from `center` (row, col) satisfy
    ``(r / radius)**2 + (c / radius)**2 < 1``, in raster order.  The bounding box runs from ceil(centre - |radius|) to
    floor(centre + |radius|), clipped to `shape` when it is given; the offsets are float, from the box's corner."""
    center = np.array(center, dtype=float)
    radius_rot = abs(radius * np.cos(0.0)) + radius * np.sin(0.0)
    upper_left = np.ceil(center - radius_rot).astype(int)
    lower_right = np.floor(center + radius_rot).astype(int)
    if shape is not None:
        upper_left = np.maximum(upper_left, np.array([0, 0]))
        lower_right = np.minimum(lower_right, np.array(shape[:2]) - 1)
    shifted = center - upper_left
    bounding = lower_right - upper_left + 1
    r_lim, c_lim = np.ogrid[0:float(bounding[0]), 0:float(bounding[1])]
    r, c = r_lim - shifted[0], c_lim - shifted[1]
    rr, cc = np.nonzero((r / radius) ** 2 + (c / radius) ** 2 < 1)
    return rr + upper_left[0], cc + upper_left[1]


def check_disk_bounds(shape: tuple[int, int], cy: float, cx: float, radius: float) -> None:
    """Raise numpy's IndexError (type and message) where ``arr[disk((cy, cx), radius)]`` would for an array of `shape`.  A bounding box
    inside [-h, h) x [-w, w) cannot raise (negative indices wrap); only a disk reaching beyond it is resolved pixel by pixel."""
    h, w = shape
    rr0, rr1 = np.ceil(cy - abs(radius)), np.floor(cy + abs(radius))
    cc0, cc1 = np.ceil(cx - abs(radius)), np.floor(cx + abs(radius))
    if rr0 >= -h and rr1 < h and cc0 >= -w and cc1 < w:
        return
    rr, cc = disk((cy, cx), radius)
    np.broadcast_to(np.uint8(0), (h, w))[rr, cc]       # numpy's own check, on a view of no memory


def disk_stats_dtype(a: np.ndarray) -> np.ndarray:
    """`a` in a dtype epid_disk_stats reads: integer and bool arrays of up to 32 bits widen to int64, whose statistics numpy forms the
    same way (every value cast to float64); float16 and 64-bit unsigned arrays raise NotImplementedError"""
    if a.dtype in nat._NP2DT:
        return a
    if a.dtype == np.bool_ or (np.issubdtype(a.dtype, np.integer) and a.dtype.itemsize <= 4):
        return a.astype(np.int64)
    raise NotImplementedError(f"disk ROI statistics of {a.dtype.name} images are not supported")


def fill_disk_stats(rois: Sequence[DiskROI], device: int | None = None) -> None:
    """Compute the statistics of every ROI of `rois` that shares the first one's array in one device call.  ROIs that would raise
    IndexError are left to raise it when read; the others keep their results, as if each had made its own call."""
    rois = [r for r in rois if r._stats is None]
    if not rois:
        return
    base = rois[0]._array
    a = np.asarray(getattr(base, "array", base))
    if a.ndim != 2:
        raise ValueError(f"a disk ROI needs a 2-D image array, got {a.ndim}-D")
    a = disk_stats_dtype(a)
    todo = []
    for r in rois:
        if r._array is not base:
            continue
        try:
            check_disk_bounds(a.shape, r.center.y, r.center.x, r.radius)
        except IndexError:
            continue
        todo.append(r)
    if not todo:
        return
    out = nat.disk_stats(nat.Context.default(device), a, [(0, r.center.y, r.center.x, r.radius) for r in todo])
    for i, r in enumerate(todo):
        r._stats = {k: float(v[i]) for k, v in out.items()}


class DiskROI(Circle):
    """A disk-shaped region of interest of an image array (or image) around `center` with `radius` pixels."""

    @classmethod
    def from_phantom_center(cls, array: np.ndarray, angle: float, roi_radius: float, dist_from_center: float,
                            phantom_center: tuple | Point):
        """The disk `dist_from_center` pixels from `phantom_center` at `angle` degrees (clockwise on screen from +x)."""
        center = cls._get_shifted_center(angle, dist_from_center, phantom_center)
        return cls(array=array, center=center, radius=roi_radius)

    def __init__(self, array: np.ndarray, radius: float, center: Point):
        super().__init__(center_point=center, radius=radius)
        self._array = array
        self._stats = None

    @staticmethod
    def _get_shifted_center(angle: float, dist_from_center: float, phantom_center: Point) -> Point:
        """The center of the ROI; corrects for phantom dislocation and roll."""
        y_shift = np.sin(np.deg2rad(angle)) * dist_from_center
        x_shift = np.cos(np.deg2rad(angle)) * dist_from_center
        return Point(phantom_center.x + x_shift, phantom_center.y + y_shift)

    def _frame(self) -> np.ndarray:
        return np.asarray(getattr(self._array, "array", self._array))

    def _stat(self, name: str) -> float:
        """one statistic from the ROI's device call (made on first use); an empty disk gives numpy's own result, warning or error"""
        if self._stats is None:
            check_disk_bounds(self._frame().shape, self.center.y, self.center.x, self.radius)
            fill_disk_stats([self])
        if self._stats["count"] == 0:
            empty = np.empty(0, self._frame().dtype)
            return float({"median": np.median, "mean": np.mean, "std": np.std, "min": np.min, "max": np.max}[name](empty))
        return self._stats[name]

    @cached_property
    def pixel_values(self) -> np.ndarray:
        return self.circle_mask()

    @cached_property
    def pixel_value(self) -> float:
        """The median pixel value of the ROI."""
        return self._stat("median")

    @cached_property
    def mean(self) -> float:
        """The mean value within the ROI."""
        return self._stat("mean")

    @cached_property
    def std(self) -> float:
        """The standard deviation of the pixel values."""
        return self._stat("std")

    @cached_property
    def min(self) -> float:
        """The min value within the ROI."""
        return self._stat("min")

    @cached_property
    def max(self) -> float:
        """The max value within the ROI."""
        return self._stat("max")

    def circle_mask(self) -> np.ndarray:
        """The pixel values of the ROI, in raster order (gathered on the host)."""
        rr, cc = disk((self.center.y, self.center.x), self.radius)
        return self._frame()[rr, cc]

    def masked_array(self) -> np.ndarray:
        """A 2D array the same shape as the underlying image array, with the pixels within the ROI set to their pixel values, and the
        rest set to nan."""
        a = self._frame()
        img = np.full(a.shape, np.nan, dtype=a.dtype)
        rr, cc = disk((self.center.y, self.center.x), self.radius, shape=a.shape)
        img[rr, cc] = a[rr, cc]
        return img

    def as_dict(self) -> dict:
        """Convert to dict. Useful for dataclasses/Result"""
        data = super().as_dict()
        data.update({"median": self.pixel_value, "std": self.std})
        return data


class HighContrastDiskROI(DiskROI):
    """A class for analyzing the high-contrast disks."""

    contrast_threshold: float | None

    @classmethod
    def from_phantom_center(cls, array: np.ndarray, angle: float, roi_radius: float, dist_from_center: float,
                            phantom_center: tuple | Point, contrast_threshold: float):
        center = cls._get_shifted_center(angle, dist_from_center, phantom_center)
        return cls(array=array, radius=roi_radius, center=center, contrast_threshold=contrast_threshold)

    def __init__(self, array: np.ndarray, radius: float, center: Point, contrast_threshold: float):
        super().__init__(array=array, radius=radius, center=center)
        self.contrast_threshold = contrast_threshold

    def __repr__(self):
        return f"High-Contrast Disk; max pixel: {self.max}, min pixel: {self.min}"


class RectangleROI(Rectangle):
    def __init__(self, array: np.ndarray, width: float, height: float, center, rotation: float = 0.0):
        if width < 2:
            raise ValueError(f"The width must be >= 2. Given {width}")
        if height < 2:
            raise ValueError(f"The height must be >= 2. Given {height}")
        super().__init__(width, height, center, rotation=rotation)
        self._array = array
        self._stats = None

    @classmethod
    def from_phantom_center(cls, array, width: float, height: float, angle: float, dist_from_center: float, phantom_center: Point,
                            rotation: float = 0.0):
        """core/roi.py:484-531"""
        y_shift = np.sin(np.deg2rad(angle)) * dist_from_center
        x_shift = np.cos(np.deg2rad(angle)) * dist_from_center
        return cls(array=array, width=width, height=height, center=Point(phantom_center.x + x_shift, phantom_center.y + y_shift),
                   rotation=rotation)

    def _polygon_xy(self) -> np.ndarray:
        """The corner list ``pixels_flat`` hands to skimage.draw.polygon (core/roi.py:646-656), as (x, y) pairs."""
        bl, br, tr, tl = self.bl_corner, self.br_corner, self.tr_corner, self.tl_corner
        return np.array([(bl.x, bl.y - 1), (br.x - 1, br.y - 1), (tr.x - 1, tr.y), (tl.x, tl.y)], dtype=np.float64)

    def _compute(self) -> dict:
        if self._stats is None:
            a = np.asarray(getattr(self._array, "array", self._array))
            if a.dtype not in nat._NP2DT:
                a = a.astype(np.float64)
            out = nat.roi_stats(nat.Context.default(), a, self._polygon_xy()[None])
            self._stats = {k: float(v[0, 0]) for k, v in out.items()}
        return self._stats

    @property
    def pixel_array(self) -> np.ndarray:
        if self.rotation != 0:
            raise ValueError("The pixel array cannot be reshaped into a 2D array when the rotation is not 0.")
        a = getattr(self._array, "array", self._array)
        return a[int(np.round(self.tl_corner.y)): int(np.round(self.bl_corner.y)), int(np.round(self.bl_corner.x)): int(np.round(self.br_corner.x))]

    @property
    def pixel_value(self) -> float:
        return self._compute()["mean"]

    @property
    def mean(self) -> float:
        return self._compute()["mean"]

    @property
    def std(self) -> float:
        return self._compute()["std"]

    @property
    def min(self) -> float:
        return self._compute()["min"]

    @property
    def max(self) -> float:
        return self._compute()["max"]

    def __repr__(self):
        return f"Rectangle ROI @ {self.center}; mean pixel: {self.pixel_value}"
