"""``DiskROI``, ``LowContrastDiskROI``, ``HighContrastDiskROI`` (core/roi.py:39-478) and ``RectangleROI`` (core/roi.py:481-706): regions of an image
array and the statistics of their pixels.

A disk's pixels are ``arr[skimage.draw.disk((cy, cx), r)]`` in the reference.  Its median, mean, std, min and max come from one
device call (``epid_disk_stats``, csrc/roi.cu), equal bit for bit to numpy's over the same pixels in the same order, and a low-contrast
disk's percentiles from another (``epid_disk_percentiles``); ``pixel_values``,
``circle_mask`` and ``masked_array`` gather on the host.  The pixel selection of a rectangle is skimage.draw.polygon's in the reference
(``pixels_flat``); here the statistics are device reductions over the same pixel set (``epid_roi_stats``, csrc/roi.cu: integer pixel
coordinates inside or on the boundary of the corner polygon the reference builds, clipped to the image).  ``pixel_array`` (non-rotated
ROIs) is a numpy view like the reference's."""
from __future__ import annotations

from collections.abc import Sequence
from functools import cached_property

import numpy as np

from .. import _native as nat
from .contrast import RMS_RANGE_MESSAGE, Contrast, contrast, michelson, ratio, rms, visibility, weber
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


def fill_disk_percentiles(rois: Sequence[LowContrastDiskROI], q: Sequence[float], device: int | None = None) -> None:
    """Compute percentiles `q` (Python numbers) of every ROI of `rois` that shares the first one's array in one device call, as
    ``roi.percentile`` reads them.  ROIs that would raise IndexError, and empty ROIs, are left to raise when read; an out-of-range q
    raises numpy's ValueError here."""
    q = list(dict.fromkeys(q))
    rois = [r for r in rois if any(x not in r._percentiles for x in q)]
    if not rois:
        return
    base = rois[0]._array
    frame = rois[0]._frame()
    if frame.dtype == np.int8:
        # numpy forms b - a in int8, wrapping, which the widened int64 copy would not
        raise NotImplementedError("disk ROI percentiles of int8 images are not supported")
    for x in q:
        # numpy's own check of q, in the type it plans in; for bool pixels numpy's TypeError (it cannot form b - a)
        np.percentile(np.zeros(1, frame.dtype), x)
    fill_disk_stats(rois, device)
    a = disk_stats_dtype(frame)
    todo = [r for r in rois if r._array is base and r._stats is not None and r._stats["count"] > 0]
    if not todo:
        return
    out = nat.disk_percentiles(nat.Context.default(device), a, [(0, r.center.y, r.center.x, r.radius) for r in todo], q)
    for i, r in enumerate(todo):
        r._percentiles.update(zip(q, out[i].tolist()))


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


class LowContrastDiskROI(DiskROI):
    """A low-contrast disk: its median against a reference value (``contrast_reference``, typically the background's median) by
    ``contrast_method``, its contrast-to-noise ratio and the Rose visibility.  ``percentile`` is numpy's over the disk's pixels, from the
    device."""

    contrast_threshold: float | None
    cnr_threshold: float | None
    contrast_reference: float | None

    @classmethod
    def from_phantom_center(cls, array: np.ndarray, angle: float, roi_radius: float, dist_from_center: float,
                            phantom_center: tuple | Point, contrast_threshold: float | None = None,
                            contrast_reference: float | None = None, cnr_threshold: float | None = None,
                            contrast_method: str = Contrast.MICHELSON, visibility_threshold: float | None = 0.1):
        center = cls._get_shifted_center(angle, dist_from_center, phantom_center)
        return cls(array=array, radius=roi_radius, center=center, contrast_threshold=contrast_threshold,
                   contrast_reference=contrast_reference, cnr_threshold=cnr_threshold, contrast_method=contrast_method,
                   visibility_threshold=visibility_threshold)

    def __init__(self, array: np.ndarray, radius: float, center: Point, contrast_threshold: float | None = None,
                 contrast_reference: float | None = None, cnr_threshold: float | None = None,
                 contrast_method: str = Contrast.MICHELSON, visibility_threshold: float = 0.1):
        super().__init__(array, radius, center=center)
        self.contrast_threshold = contrast_threshold
        self.cnr_threshold = cnr_threshold
        self.contrast_reference = contrast_reference
        self.contrast_method = contrast_method
        self.visibility_threshold = visibility_threshold
        self._percentiles = {}

    @property
    def _contrast_array(self) -> np.ndarray:
        return np.array((self.pixel_value, self.contrast_reference))

    @property
    def signal_to_noise(self) -> float:
        """The median over the std, divided as numpy divides (a zero std gives inf or nan and numpy's warning)."""
        return float(np.array(self.pixel_value) / self.std)

    @property
    def contrast_to_noise(self) -> float:
        """The contrast over the std, divided as numpy divides."""
        return float(np.array(self.contrast) / self.std)

    @property
    def michelson(self) -> float:
        return michelson(self._contrast_array)

    @property
    def weber(self) -> float:
        return weber(feature=self.pixel_value, background=self.contrast_reference)

    @property
    def rms(self) -> float:
        return rms(self._contrast_array)

    @property
    def ratio(self) -> float:
        return ratio(self._contrast_array)

    @property
    def contrast(self) -> float:
        """The contrast of the median against ``contrast_reference`` by ``contrast_method``."""
        return contrast(self._contrast_array, self.contrast_method)

    @property
    def cnr_constant(self) -> float:
        """The contrast-to-noise ratio times the diameter (superseded by ``visibility``)."""
        return self.contrast_to_noise * self.diameter

    @property
    def visibility(self) -> float:
        """The Rose model's visibility of the disk (core.contrast.visibility)."""
        return visibility(array=self._contrast_array, radius=self.radius, std=self.std, algorithm=self.contrast_method)

    @property
    def contrast_constant(self) -> float:
        """The contrast times the diameter (superseded by ``visibility``)."""
        return self.contrast * self.diameter

    @property
    def passed(self) -> bool:
        return self.contrast > self.contrast_threshold

    @property
    def passed_visibility(self) -> bool:
        return self.visibility > self.visibility_threshold

    @property
    def passed_contrast_constant(self) -> bool:
        return self.contrast_constant > self.contrast_threshold

    @property
    def passed_cnr_constant(self) -> bool:
        return self.cnr_constant > self.cnr_threshold

    @property
    def plot_color(self) -> str:
        return "green" if self.passed_visibility else "red"

    @property
    def plot_color_constant(self) -> str:
        return "green" if self.passed_contrast_constant else "red"

    @property
    def plot_color_cnr(self) -> str:
        return "green" if self.passed_cnr_constant else "red"

    def as_dict(self) -> dict:
        return {
            "contrast method": self.contrast_method,
            "visibility": self.visibility,
            "visibility threshold": self.visibility_threshold,
            "passed visibility": bool(self.passed_visibility),
            "contrast": self.contrast,
            "cnr": self.contrast_to_noise,
            "signal to noise": self.signal_to_noise,
        }

    def percentile(self, percentile: float) -> float:
        """``np.percentile`` of the ROI's pixels (method "linear") for a Python number `percentile`, from the device; an empty ROI,
        a disk beyond the frame and an out-of-range percentile raise numpy's exceptions."""
        if percentile not in self._percentiles:
            check_disk_bounds(self._frame().shape, self.center.y, self.center.x, self.radius)
            if self._frame().dtype == np.bool_:
                np.percentile(self.circle_mask(), percentile)   # always raises for bool pixels, as in the reference
            fill_disk_percentiles([self], [percentile])
            if self._stats["count"] == 0:
                return float(np.percentile(np.empty(0, self._frame().dtype), percentile))
        return self._percentiles[percentile]


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


class LowContrastFrame:
    """The low-contrast analysis of one frame of analyze_low_contrast_batch, as ``ImagePhantomBase`` computes it from its
    ``LowContrastDiskROI``s: the ``background`` value (np.mean of the background disks' medians) and, per low-contrast disk in the
    settings' order, lists of ``centers``, ``radii``, ``medians``, ``stds``, ``contrasts``, ``cnrs`` (contrast to noise),
    ``snrs`` (signal to noise), ``visibilities``, ``passed_visibility`` and ``percentiles`` (one pair per disk), and ``piu``, the
    lowest percent integral uniformity of the disks.  An empty disk or one with a NaN pixel gives NaN where the reference raises or warns."""

    def __init__(self, **fields):
        self.__dict__.update(fields)

    @property
    def passed(self) -> list[bool]:
        """each disk's contrast above ``contrast_threshold`` (None raises TypeError, as in the reference)"""
        return [c > self.contrast_threshold for c in self.contrasts]


def _per_frame(value, n: int, name: str, width: int | None = None) -> list:
    """a scalar geometry value repeated n times, or the n entries of a per-frame one; with `width`, a value is a Point or `width`
    numbers, and a per-frame one n of either"""
    if width is not None:
        if isinstance(value, Point):
            return [value] * n
        if not isinstance(value, np.ndarray) and any(isinstance(v, Point) for v in value):
            value = [(v.x, v.y) if isinstance(v, Point) else v for v in value]
    a = np.asarray(value, dtype=np.float64)
    if a.ndim == (0 if width is None else 1):
        return [value] * n
    if a.shape[0] != n:
        raise ValueError(f"{name} has {a.shape[0]} entries for {n} frames")
    return a.tolist()


def _batch_contrast(method: str, m: np.ndarray, bg: np.ndarray) -> np.ndarray:
    """contrast(np.array((median, background)), method) for every disk at once, in the same float64 operations"""
    key = method.lower()
    if key == Contrast.MICHELSON.lower():
        hi, lo = np.fmax(m, bg), np.fmin(m, bg)           # np.nanmax / np.nanmin of the pair
        return (hi - lo) / (hi + lo)
    if key == Contrast.WEBER.lower():
        return np.abs(m - bg) / bg
    if key == Contrast.RATIO.lower():
        return m / bg
    if key == Contrast.DIFFERENCE.lower():
        return np.abs(m - bg)
    if key == Contrast.RMS.lower():
        if np.any((np.minimum(m, bg) < 0) | (np.maximum(m, bg) > 1)):
            raise ValueError(RMS_RANGE_MESSAGE)
        mu = (m + bg) / 2
        return np.sqrt(((m - mu) ** 2 + (bg - mu) ** 2) / 2)
    return contrast(np.zeros(2), method)                 # the reference's ValueError for an unknown method


def analyze_low_contrast_batch(frames, phantom_center, phantom_angle, phantom_radius, low_contrast_rois: dict, background_rois: dict, *,
                               contrast_method: str = Contrast.MICHELSON, contrast_threshold: float | None = None,
                               visibility_threshold: float = 0.1, roi_size_factor: float = 1.0, percentiles=(1, 99),
                               device: int | None = None) -> list[LowContrastFrame]:
    """The low-contrast stage of the planar image-quality phantoms (``ImagePhantomBase._sample_low_contrast_background_rois``,
    ``_sample_low_contrast_rois`` and ``percent_integral_uniformity``) for every frame of `frames` (an [n, h, w] or [h, w] ndarray or a
    device Batch) whose phantom geometry is known: `phantom_center` (a Point or (x, y), or n of them), `phantom_angle` (degrees) and
    `phantom_radius` (pixels), each a scalar or one per frame.  The ROI settings use the reference's keys ("angle", "distance from
    center", "roi radius").  The statistics of all disks of all frames come from one ``epid_disk_stats`` call and the percentiles of all
    low-contrast disks from one ``epid_disk_percentiles`` call; a disk beyond a frame raises numpy's IndexError first.  Every value
    equals the reference's bit for bit."""
    if isinstance(frames, nat.Batch):
        (n, h, w), dtype = frames.shape_dtype
    else:
        frames = np.asarray(frames)
        frames = frames[None] if frames.ndim == 2 else frames
        if frames.ndim != 3:
            raise ValueError(f"frames must be [n, h, w] or [h, w], got {frames.ndim}-D")
        dtype = frames.dtype
        frames = disk_stats_dtype(frames)
        n, h, w = frames.shape
    if np.dtype(dtype) == np.int8:
        raise NotImplementedError("disk ROI percentiles of int8 images are not supported")
    percentiles = list(percentiles)
    if len(percentiles) != 2:
        raise ValueError("percentiles must be a (low, high) pair")
    for x in percentiles:
        np.percentile(np.zeros(1, dtype), x)
    centers = [c if isinstance(c, Point) else Point(*c) for c in _per_frame(phantom_center, n, "phantom_center", 2)]
    angles = _per_frame(phantom_angle, n, "phantom_angle")
    radii = _per_frame(phantom_radius, n, "phantom_radius")

    geometry = {}                                        # (centre, angle, radius) -> (bg disks, lc disks) as (cy, cx, r)
    rows_bg, rows_lc, frame_disks = [], [], []
    for f in range(n):
        key = (centers[f].x, centers[f].y, angles[f], radii[f])
        if key not in geometry:
            def place(settings, rad=radii[f], ang=angles[f], c=centers[f]):
                out = []
                for st in settings.values():
                    p = DiskROI._get_shifted_center(ang + st["angle"], rad * st["distance from center"], c)
                    r = rad * st["roi radius"] * roi_size_factor
                    check_disk_bounds((h, w), p.y, p.x, r)
                    out.append((p.y, p.x, r))
                return out
            geometry[key] = (place(background_rois), place(low_contrast_rois))
        bg, lc = geometry[key]
        rows_bg += [(f, *d) for d in bg]
        rows_lc += [(f, *d) for d in lc]
        frame_disks.append(lc)
    nbg, nlc = len(background_rois), len(low_contrast_rois)
    ctx = nat.Context.default(device)
    stats = nat.disk_stats(ctx, frames, rows_bg + rows_lc)
    pct = nat.disk_percentiles(ctx, frames, rows_lc, percentiles) if rows_lc else np.zeros((0, len(percentiles)))
    med_bg = stats["median"][:n * nbg].reshape(n, nbg)
    med = stats["median"][n * nbg:].reshape(n, nlc)
    std = stats["std"][n * nbg:].reshape(n, nlc)
    pct = pct.reshape(n, nlc, len(percentiles))
    background = np.array([np.mean(med_bg[f].tolist()) for f in range(n)])
    sqrt_area = np.array([[np.sqrt(r**2 * np.pi) for (_, _, r) in frame_disks[f]] for f in range(n)]).reshape(n, nlc)
    with np.errstate(all="ignore"):
        con = _batch_contrast(contrast_method, med, background[:, None])
        vis = con * sqrt_area / std
        cnr, snr = con / std, med / std
        lo, hi = pct[:, :, 0], pct[:, :, 1]
        piu = 100 * (1 - (hi - lo + 1e-6) / (hi + lo + 1e-6))
    out = []
    for f in range(n):
        out.append(LowContrastFrame(
            background=float(background[f]), centers=[Point(x, y) for (y, x, _) in frame_disks[f]],
            radii=[r for (_, _, r) in frame_disks[f]], medians=med[f].tolist(), stds=std[f].tolist(), contrasts=con[f].tolist(),
            cnrs=cnr[f].tolist(), snrs=snr[f].tolist(), visibilities=vis[f].tolist(),
            passed_visibility=(vis[f] > visibility_threshold).tolist(), percentiles=pct[f].tolist(),
            piu=min(piu[f].tolist()) if nlc else None, contrast_method=contrast_method, contrast_threshold=contrast_threshold,
            visibility_threshold=visibility_threshold))
    return out
