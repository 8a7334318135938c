"""pylinac.nuclear (nuclear.py:39-500, 1370-1856): MaxCountRate, PlanarUniformity, TomographicUniformity and TomographicContrast of
gamma-camera NM files.

PlanarUniformity's whole frame pipeline (binning, the NEMA 9-point filter, the threshold, the stray-pixel clean-up, the largest
component, both FOV erosions, integral and differential uniformity) runs in one device call per batch (csrc/nuclear.cu), bit-identical
to the reference.  The cleaned frames and FOV masks stay on the device until an attribute needs them.  MaxCountRate takes its exact
frame sums from epid_frame_stats.  TomographicContrast makes one device call for the slice analysis of a batch of SPECT volumes and
one for all its sphere searches (csrc/nuclear_tomo.cu), bit-identical to the reference.  TomographicUniformity averages a slab of
slices and runs the planar pipeline on that float64 frame, with a third (center) FOV, in one device call per batch
(csrc/nuclear_tu.cu), bit-identical to the reference.  QuadrantResolution takes the mean and standard deviation of four disk ROIs
from one device call (epid_disk_stats, csrc/roi.cu), equal bit for bit to numpy's, and forms the moments MTF on the host in the
reference's expressions.  The other nuclear tests are not ported yet (DESIGN.md section 6).
"""
from __future__ import annotations

import json
import math
import warnings
from collections.abc import Sequence
from functools import cached_property
from pathlib import Path
from typing import TypedDict

import numpy as np
from pydantic import BaseModel

from . import _native as nat
from .core.geometry import Point, direction_to_coords
from .core.image import NMImageStack
from .core.mtf import MomentMTF
from .core.roi import HighContrastDiskROI, check_disk_bounds, disk_stats_dtype, fill_disk_stats
from .core.utilities import ResultBase, ResultsDataMixin
from .core.warnings import capture_warnings

# the reference's messages where it raises (Python's max() of nothing, numpy's empty reduction / all-nan argmax, sliding_window_view)
_EMPTY_MAX = "max() iterable argument is empty"
_EMPTY_FOV = "zero-size array to reduction operation fmax which has no identity"
_ALL_NAN = "All-NaN slice encountered"
_WINDOW_TOO_LARGE = "window shape cannot be larger than input array shape"


def determine_binning(pixel_size: float) -> int:
    """The block size, a power of two, that first brings `pixel_size` (mm) up to at least 4.48 mm, the lower end of NEMA's
    4.48-8.32 mm range."""
    binning = 1
    while pixel_size < 4.48:
        pixel_size *= 2
        binning *= 2
    return binning


def integral_uniformity(array: np.ndarray) -> float:
    """(max - min) / (max + min) x 100 of `array`, nan values ignored: the IAEA NMQC integral uniformity."""
    l_max, l_min = np.nanmax(array), np.nanmin(array)
    return (l_max - l_min) / (l_max + l_min) * 100


def _inner_boundary(mask: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """find_boundaries(mask, connectivity=1, mode="inner") as (boundary_x, boundary_y): the mask pixels with a 4-neighbour outside
    the mask; beyond the frame edge a pixel is its own neighbour."""
    m = np.asarray(mask, dtype=bool)
    p = np.pad(m, 1, mode="edge")
    inner = p[:-2, 1:-1] & p[2:, 1:-1] & p[1:-1, :-2] & p[1:-1, 2:]
    by, bx = np.nonzero(m & ~inner)
    return bx, by


def get_fov(array: np.ndarray, size: float) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(fov_array, boundary_x, boundary_y) of the UFOV or CFOV of `array`, `size` being the FOV's fraction of the longest side.

    The largest 4-connected component of ``array > 0`` sets the erosion ``int(round((1 - size) * longest side))``; the FOV is every
    pixel whose Euclidean distance to the background exceeds half of it.  Runs on the device (epid_nm_fov).
    """
    array = np.asarray(array)
    if array.ndim != 2:
        raise ValueError(f"get_fov takes a 2-D array, got {array.ndim}-D")
    row, mask = nat.nm_fov(nat.Context.default(), array > 0, 1 - size)
    if row["status"] == nat.NM_NO_COMPONENT:
        raise ValueError(_EMPTY_MAX)
    eroded = mask.astype(bool)
    bx, by = _inner_boundary(eroded)
    return np.where(eroded, array, 0), bx, by


class _DeviceArrays:
    """The cleaned frames and FOV masks of one analyze_batch call, on the device until first read, then downloaded once."""

    def __init__(self, cleaned: nat.Batch | None, masks: nat.Batch | None, mean: nat.Batch | None = None):
        self._batches = {"cleaned": cleaned, "masks": masks, "mean": mean}
        self._host = {}

    def get(self, name: str) -> np.ndarray:
        if name not in self._host:
            b = self._batches[name]
            if b is None:
                raise RuntimeError("analyze_batch(arrays=False) keeps no frame arrays")
            self._host[name] = b.download()
            b.free()
        return self._host[name]


class FOV:
    """A field of view (UFOV or CFOV) of one analysed frame (nuclear.py:158-271): the uniformities are read from the device row, the
    arrays are downloaded on first access.  Unlike the reference's dataclass it is built by the analysis from a device row, not from
    a FOV array."""

    _masks_per_frame = 2           # the masks batch holds this many masks per frame, FOV k of frame f at f * _masks_per_frame + k

    def __init__(self, name: str, window_size: int, row, k: int, shape: tuple[int, int], arrays: _DeviceArrays, frame: int):
        self.name = name
        self.window_size = window_size
        self._row, self._k, self._shape, self._arrays, self._frame = row, k, shape, arrays, frame

    @property
    def mask(self) -> np.ndarray:
        """the eroded binary of the frame (bool)"""
        return self._arrays.get("masks")[self._masks_per_frame * self._frame + self._k].astype(bool)

    @property
    def fov(self) -> np.ndarray:
        return np.where(self.mask, self._arrays.get("cleaned")[self._frame], 0)

    @property
    def boundary_x(self) -> np.ndarray:
        return _inner_boundary(self.mask)[0]

    @property
    def boundary_y(self) -> np.ndarray:
        return _inner_boundary(self.mask)[1]

    @property
    def erosion(self) -> int:
        """int(round((1 - size) * longest side of the largest component))"""
        return int(self._row["erosion"][self._k])

    @property
    def integral_uniformity(self) -> float:
        """integral uniformity (%) of the non-zero FOV pixels"""
        if self._row["n_fov"][self._k] == 0:
            raise ValueError(_EMPTY_FOV)
        return float(self._row["iu"][self._k])

    def _axis_max(self, axis: int) -> tuple[float, tuple[int, int]]:
        """(max window uniformity, first (i, j) of it) of the windows along `axis`"""
        if self.window_size > self._shape[0] or self.window_size > self._shape[1]:
            raise ValueError(_WINDOW_TOO_LARGE)
        j = 2 * self._k + axis
        if self._row["du_count"][j] == 0:
            raise ValueError(_EMPTY_MAX)
        pos = int(self._row["du_index"][j])
        return float(self._row["du_max"][j]), (pos // self._shape[1], pos % self._shape[1])

    @property
    def differential_uniformity_x(self) -> tuple[float, tuple[int, int]]:
        """the maximum uniformity of the windows along axis 1 and the first window position (i, j) holding it"""
        return self._axis_max(1)

    @property
    def differential_uniformity_y(self) -> tuple[float, tuple[int, int]]:
        """the maximum uniformity of the windows along axis 0 and the first window position (i, j) holding it"""
        return self._axis_max(0)

    @property
    def differential_uniformity(self) -> float:
        """the largest window uniformity (%) along either axis"""
        self._axis_max(0)                          # the reference builds the axis-0 windows first
        return max(self._axis_max(1)[0], self._axis_max(0)[0])

    def _point(self, key: str) -> tuple[int, int]:
        if self._row["n_fov"][self._k] == 0:
            raise ValueError(_ALL_NAN)
        idx = int(self._row[key][self._k])
        return idx // self._shape[1], idx % self._shape[1]

    @property
    def max_point(self) -> tuple[int, int]:
        """(row, col) of the first FOV maximum in raster order"""
        return self._point("max_index")

    @property
    def min_point(self) -> tuple[int, int]:
        """(row, col) of the first FOV minimum in raster order"""
        return self._point("min_index")


class UniformityFrame:
    """One frame of analyze_batch: ``ufov``, ``cfov`` (FOV), ``binned_frame`` (the cleaned float64 frame) and the device row."""

    def __init__(self, row, window_size: int, shape: tuple[int, int], arrays: _DeviceArrays, frame: int):
        self.row = row
        self._arrays, self._frame = arrays, frame
        self.ufov = FOV("UFOV", window_size, row, 0, shape, arrays, frame)
        self.cfov = FOV("CFOV", window_size, row, 1, shape, arrays, frame)

    @property
    def status(self) -> int:
        return int(self.row["status"])

    @property
    def longest_side(self) -> int:
        """the longest bounding-box side of the largest component"""
        return int(self.row["longest"])

    def raise_for_status(self) -> None:
        """get_fov's ValueError for a frame with no component left after the clean-up"""
        if self.status == nat.NM_NO_COMPONENT:
            raise ValueError(_EMPTY_MAX)

    @property
    def binned_frame(self) -> np.ndarray:
        return self._arrays.get("cleaned")[self._frame]


class UniformityBatchResult(Sequence):
    def __init__(self, rows: np.ndarray, bin_size: int, window_size: int, shape: tuple[int, int], arrays: _DeviceArrays):
        self.rows = rows
        self.bin_size = bin_size
        self.window_size = window_size
        self.shape = shape
        self._arrays = arrays

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, i) -> UniformityFrame:
        return UniformityFrame(self.rows[i], self.window_size, self.shape, self._arrays, range(len(self.rows))[i])


def analyze_batch(frames, pixel_size_mm: float, *, ufov_ratio: float = 0.95, cfov_ratio: float = 0.75, window_size: int = 5,
                  threshold: float = 0.75, arrays: bool = True, device: int | None = None) -> UniformityBatchResult:
    """``PlanarUniformity.analyze(ufov_ratio, cfov_ratio, window_size, threshold)`` for every frame of `frames` (uint16 [n, h, w]
    ndarray or device Batch; uint8 is widened on the host) in one device call.  `arrays`: keep each frame's cleaned frame and FOV masks
    on the device for ``binned_frame`` / ``fov`` / ``boundary_*``.  Rows raise the reference's exceptions from
    ``raise_for_status()`` and the FOV properties."""
    if int(window_size) != window_size or window_size < 1:
        raise ValueError(f"window_size must be a positive integer, got {window_size}")
    ctx = nat.Context.default(device)
    if isinstance(frames, nat.Batch):
        (_, h, w), dt = frames.shape_dtype
        if dt != np.uint16:
            raise NotImplementedError(f"nuclear frames of dtype {np.dtype(dt).name} are not supported (uint8 or uint16)")
    else:
        a = np.asarray(frames)
        if a.dtype == np.uint8:
            a = a.astype(np.uint16)
        elif a.dtype != np.uint16:
            raise NotImplementedError(f"nuclear frames of dtype {a.dtype.name} are not supported (uint8 or uint16)")
        frames = a[None] if a.ndim == 2 else a
        h, w = frames.shape[1:]
    b = determine_binning(pixel_size_mm)
    # the reference's own expressions: 1 - size with size = cfov_ratio * ufov_ratio for the CFOV
    rows, cleaned, masks = nat.nm_uniformity(ctx, frames, b, 1 - ufov_ratio, 1 - cfov_ratio * ufov_ratio, int(window_size), threshold,
                                             arrays=arrays)
    return UniformityBatchResult(rows, b, int(window_size), (-(-h // b), -(-w // b)), _DeviceArrays(cleaned, masks))


class PlanarUniformityResults(BaseModel):
    ufov_integral_uniformity: float  #:
    ufov_differential_uniformity: float  #:
    cfov_integral_uniformity: float  #:
    cfov_differential_uniformity: float  #:


class PlanarUniformity:
    """NEMA integral and differential uniformity of every frame of an NM flood file (nuclear.py:274-396)."""

    stack: NMImageStack
    frame_results: dict

    def __init__(self, path: str | Path) -> None:
        self.stack = NMImageStack(path)
        self.path = Path(path)

    def analyze(self, ufov_ratio: float = 0.95, cfov_ratio: float = 0.75, window_size: int = 5, threshold: float = 0.75) -> None:
        """Uniformities of the UFOV (`ufov_ratio` of the detected field) and the CFOV (`cfov_ratio` of the UFOV) of every frame,
        with differential windows of `window_size` binned pixels; pixels below `threshold` x the mean of those above 10 % of the
        maximum are dropped first.  Raises ValueError for the first frame with nothing left."""
        pixel_size = float(self.stack.metadata.PixelSpacing[0])
        res = analyze_batch(self.stack._pixels, pixel_size, ufov_ratio=ufov_ratio, cfov_ratio=cfov_ratio, window_size=window_size,
                            threshold=threshold)
        for r in res:
            r.raise_for_status()
        self.frame_results = {str(k + 1): {"ufov": r.ufov, "cfov": r.cfov, "binned_frame": r.binned_frame} for k, r in enumerate(res)}

    def results(self) -> str:
        """the uniformities of every frame as text"""
        s = []
        for key, result in self.frame_results.items():
            s.append(f"Frame {key}:\n")
            s.append(f"UFOV integral uniformity: {result['ufov'].integral_uniformity:.2f}%\n")
            s.append(f"UFOV differential uniformity {result['ufov'].differential_uniformity:.2f}%\n")
            s.append(f"CFOV integral uniformity: {result['cfov'].integral_uniformity:.2f}%\n")
            s.append(f"CFOV differential uniformity {result['cfov'].differential_uniformity:.2f}%\n")
            s.append("\n")
        return "".join(s)

    def results_data(self, as_dict: bool = False, as_json: bool = False) -> dict | str:
        data = {}
        for key, result in self.frame_results.items():
            r = PlanarUniformityResults(
                ufov_integral_uniformity=result["ufov"].integral_uniformity,
                ufov_differential_uniformity=result["ufov"].differential_uniformity,
                cfov_integral_uniformity=result["cfov"].integral_uniformity,
                cfov_differential_uniformity=result["cfov"].differential_uniformity,
            )
            if as_dict:
                data[f"Frame {key}"] = r.model_dump()
            elif as_json:
                data[f"Frame {key}"] = r.model_dump_json()
            else:
                data[f"Frame {key}"] = r
        if as_json:
            data = json.dumps(data)
        return data


class MaxCountRateResults(ResultBase):
    max_countrate: float  #:
    max_frame: int  #:
    frame_duration: float  #:
    sums: dict[int, float]  #:


def frame_sums(frames, device: int | None = None) -> np.ndarray:
    """exact per-frame pixel sums (float64, < 2^53) of uint8 / uint16 frames ([n, h, w] ndarray or device Batch), from epid_frame_stats"""
    ctx = nat.Context.default(device)
    if not isinstance(frames, nat.Batch):
        frames = np.asarray(frames)
        if frames.dtype not in (np.uint8, np.uint16):
            raise NotImplementedError(f"nuclear frames of dtype {frames.dtype.name} are not supported (uint8 or uint16)")
    with nat.batch_for(ctx, frames) as b:
        return nat.frame_stats(ctx, b)["sum"]


@capture_warnings
class MaxCountRate(ResultsDataMixin[MaxCountRateResults]):
    """Peak count rate of a dynamic NM acquisition (nuclear.py:46-148; IAEA NMQC test 4.2)."""

    stack: NMImageStack
    frame_duration: float
    sums: dict[int, float]

    def __init__(self, path: str | Path) -> None:
        super().__init__()
        self.stack = NMImageStack(path)

    def analyze(self, frame_duration: float = 1.0) -> None:
        """Count rate of every frame: its exact pixel sum over `frame_duration` seconds."""
        self.frame_duration = frame_duration
        self.sums = {idx: s / frame_duration for idx, s in enumerate(frame_sums(self.stack._pixels))}

    @property
    def max_countrate(self) -> float:
        """highest count rate, counts per second"""
        return max(self.sums.values())

    @property
    def max_frame(self) -> int:
        """0-based index of the first frame with the highest count rate"""
        return max(self.sums, key=self.sums.get)

    @property
    def max_time(self) -> float:
        """start time (s) of that frame"""
        return self.max_frame * self.frame_duration

    def results(self) -> str:
        """the peak count rate, frame duration and peak frame as text"""
        return (
            f"Max countrate: {self.max_countrate:.0f} counts/second\n"
            f"Frame duration: {self.frame_duration:.2f} seconds\n"
            f"Max frame: {self.max_frame} out of {len(self.stack.frames)}\n"
        )

    def _generate_results_data(self) -> MaxCountRateResults:
        return MaxCountRateResults(max_countrate=self.max_countrate, frame_duration=self.frame_duration, max_frame=self.max_frame,
                                   sums=self.sums)


# ---------------------------------------------------------------------------------------------------- TomographicUniformity
_EMPTY_MEAN_DOT = "Mean of empty slice."
_INVALID_DIVIDE = "invalid value encountered in divide"
_INVALID_SCALAR_DIVIDE = "invalid value encountered in scalar divide"


def _slab(n: int, first_frame: int, last_frame: int) -> tuple[int, int]:
    """TomographicUniformity.analyze's frame checks, in the reference's expressions and order: the slab [first, last) of n slices,
    which is empty when last is 0"""
    if first_frame < 0:
        raise ValueError("The first frame index is outside the array bounds. Increase the first frame index.")
    if last_frame < 0:
        last_frame += n
    if last_frame >= n:
        raise ValueError("The last frame index is outside the array bounds. Decrease the last frame index.")
    if 0 < last_frame <= first_frame:
        raise ValueError("The first frame index must be less than the last frame index.")
    return first_frame, last_frame


def _warn_empty_slab() -> None:
    """the warnings of the reference on an empty slab: mean(axis=0) of no slice, then preprocess's mean of an empty selection"""
    warnings.warn(_EMPTY_MEAN_DOT, RuntimeWarning, stacklevel=3)
    warnings.warn(_INVALID_DIVIDE, RuntimeWarning, stacklevel=3)
    _warn_empty_threshold()


def _warn_empty_threshold() -> None:
    """preprocess's ``array[array > max * 0.10].mean()`` of an empty selection"""
    warnings.warn(_EMPTY_MEAN_DOT, RuntimeWarning, stacklevel=4)
    warnings.warn(_INVALID_SCALAR_DIVIDE, RuntimeWarning, stacklevel=4)


class _SlabFOV(FOV):
    """A FOV of TomographicUniformity: three masks per volume (UFOV, CFOV, center), and the reference's "All-NaN slice encountered"
    warnings, two per all-nan window (nanmax, nanmin), emitted from the device row's window counts on the first differential-uniformity
    access (the reference caches the window loop).  The center FOV's ``fov`` is nan where it is 0, as center_border_ratio leaves it."""

    _masks_per_frame = 3

    def __init__(self, *args, nan_zeros: bool = False, **kwargs):
        super().__init__(*args, **kwargs)
        self._nan_zeros = nan_zeros
        self._windows_done = False

    @property
    def fov(self) -> np.ndarray:
        a = super().fov
        return np.where(a == 0, np.nan, a) if self._nan_zeros else a

    def _axis_max(self, axis: int) -> tuple[float, tuple[int, int]]:
        if not self._windows_done and not (self.window_size > self._shape[0] or self.window_size > self._shape[1]):
            self._windows_done = True
            hb, wb = self._shape
            totals = ((hb - self.window_size + 1) * wb, hb * (wb - self.window_size + 1))     # the y windows first, then x
            for a in (0, 1):
                for _ in range(2 * (totals[a] - int(self._row["du_count"][2 * self._k + a]))):
                    warnings.warn(_ALL_NAN, RuntimeWarning, stacklevel=4)
        return super()._axis_max(axis)


def _center_border_ratio(row) -> np.float64:
    """np.nanmean(center) / np.nanmean(ring) from the exact-order sums and counts of the device row"""
    means = []
    for key in ("center", "ring"):
        n = int(row[f"{key}_count"])
        if n == 0:
            warnings.warn(_EMPTY_MEAN, RuntimeWarning, stacklevel=3)
            means.append(np.float64(np.nan))
        else:
            means.append(np.float64(row[f"{key}_sum"]) / np.float64(n))
    return means[0] / means[1]


class TomographicUniformityVolume:
    """One volume of analyze_tomographic_uniformity_batch: ``row`` (the device's TU_RESULT_DTYPE row), ``ufov``, ``cfov`` and
    ``center_fov`` (FOV), ``center_border_ratio``, ``binned_frame`` (the cleaned float64 frame) and ``mean_frame`` (the slab mean)."""

    def __init__(self, row, window_size: int, shape: tuple[int, int], arrays: _DeviceArrays, volume: int):
        self.row = row
        self._arrays, self._volume = arrays, volume
        self.ufov = _SlabFOV("UFOV", window_size, row, 0, shape, arrays, volume)
        self.cfov = _SlabFOV("CFOV", window_size, row, 1, shape, arrays, volume)
        self.center_fov = _SlabFOV("Center", window_size, row, 2, shape, arrays, volume, nan_zeros=True)

    @property
    def status(self) -> int:
        return int(self.row["status"])

    def raise_for_status(self) -> None:
        """get_fov's ValueError for a volume with no component left after the clean-up"""
        if self.status == nat.NM_NO_COMPONENT:
            raise ValueError(_EMPTY_MAX)

    @property
    def center_border_ratio(self) -> np.float64:
        self.raise_for_status()
        return _center_border_ratio(self.row)

    @property
    def binned_frame(self) -> np.ndarray:
        return self._arrays.get("cleaned")[self._volume]

    @property
    def mean_frame(self) -> np.ndarray:
        return self._arrays.get("mean")[self._volume]


def _volumes(volumes, slices_per_volume):
    """(uint16 volumes as an [n, z, h, w] ndarray or a device Batch, z, h, w); uint8 widened, other dtypes NotImplementedError"""
    if isinstance(volumes, nat.Batch):
        (n, h, w), dt = volumes.shape_dtype
        if dt != np.uint16:
            raise NotImplementedError(f"nuclear frames of dtype {np.dtype(dt).name} are not supported (uint8 or uint16)")
        if slices_per_volume is None or slices_per_volume < 1 or n % slices_per_volume:
            raise ValueError(f"slices_per_volume must divide the batch's {n} slices, got {slices_per_volume}")
        return volumes, int(slices_per_volume), h, w
    a = np.asarray(volumes)
    if a.dtype == np.uint8:
        a = a.astype(np.uint16)
    elif a.dtype != np.uint16:
        raise NotImplementedError(f"nuclear frames of dtype {a.dtype.name} are not supported (uint8 or uint16)")
    if a.ndim not in (3, 4):
        raise ValueError(f"volumes must be [n, z, h, w] or [z, h, w], got {a.ndim}-D")
    a = a[None] if a.ndim == 3 else a
    return a, a.shape[1], a.shape[2], a.shape[3]


def analyze_tomographic_uniformity_batch(volumes, pixel_size_mm: float, first_frame: int = 0, last_frame: int = -1,
                                         ufov_ratio: float = 0.8, cfov_ratio: float = 0.75, center_ratio: float = 0.4,
                                         threshold: float = 0.75, window_size: int = 5, *, slices_per_volume: int | None = None,
                                         arrays: bool = True, device: int | None = None) -> list[TomographicUniformityVolume]:
    """``TomographicUniformity.analyze`` for every volume of `volumes`: a uint16 [n, z, h, w] (or [z, h, w]) ndarray, uint8 widened on
    the host, or a device Batch of n x z slices with ``slices_per_volume=z``.  The frame checks raise the reference's ValueError before
    any device call, as does an empty slab (last frame 0).  One device call analyses every volume; `arrays` keeps the slab means,
    cleaned frames and masks on the device for ``mean_frame`` / ``binned_frame`` / ``fov``."""
    if int(window_size) != window_size or window_size < 1:
        raise ValueError(f"window_size must be a positive integer, got {window_size}")
    volumes, nz, h, w = _volumes(volumes, slices_per_volume)
    first, last = _slab(nz, first_frame, last_frame)
    if last == 0:
        _warn_empty_slab()
        raise ValueError(_EMPTY_MAX)
    b = determine_binning(pixel_size_mm)
    # the reference's own expressions: 1 - size with size = cfov_ratio * ufov_ratio (CFOV) and center_ratio * ufov_ratio (center)
    erode = (1 - ufov_ratio, 1 - cfov_ratio * ufov_ratio, 1 - center_ratio * ufov_ratio)
    rows, mean, cleaned, masks = nat.tu_uniformity(nat.Context.default(device), volumes, nz, first, last - first, b, erode,
                                                   int(window_size), threshold, arrays=arrays)
    dev = _DeviceArrays(cleaned, masks, mean)
    shape = (-(-h // b), -(-w // b))
    return [TomographicUniformityVolume(r, int(window_size), shape, dev, v) for v, r in enumerate(rows)]


class _SlabMeanFrame:
    """stack.frames[0] after TomographicUniformity.analyze: the first frame's header with the slab mean as its array, downloaded from
    the device on first access"""

    def __init__(self, frame, arrays: _DeviceArrays):
        self._frame, self._arrays, self._array = frame, arrays, None

    def __getattr__(self, name):
        return getattr(self._frame, name)

    @property
    def array(self) -> np.ndarray:
        if self._array is None:
            self._array = self._arrays.get("mean")[0]
        return self._array

    @array.setter
    def array(self, value: np.ndarray) -> None:
        self._array = value


class TomographicUniformityResults(ResultBase):
    cfov_integral_uniformity: float
    cfov_differential_uniformity: float
    ufov_integral_uniformity: float
    ufov_differential_uniformity: float
    center_border_ratio: float
    first_frame: int
    last_frame: int


@capture_warnings
class TomographicUniformity(ResultsDataMixin[TomographicUniformityResults], PlanarUniformity):
    """Tomographic uniformity of a SPECT volume, typically a Jaszczak phantom (nuclear.py:1380-1551): PlanarUniformity's analysis of
    the mean of a slab of slices, and the center-to-border ratio."""

    center_ratio: float
    first_frame: int
    last_frame: int
    threshold: float

    def __init__(self, path: str | Path) -> None:
        PlanarUniformity.__init__(self, path)

    @property
    def frame_result(self) -> dict:
        """We always have a single result"""
        return self.frame_results[self.frame_key]

    @property
    def frame_key(self) -> str:
        """The key for the single frame result"""
        return f"{self.first_frame}:{self.last_frame}"

    def center_border_ratio(self, center_ratio: float, window_size: int) -> float:
        """The center-to-border ratio as defined by the NMQC toolkit: the mean of the center FOV (`center_ratio` of the phantom) over
        the mean of the border, the UFOV without the CFOV.  Stores the center FOV as ``frame_result["center_fov"]``."""
        vol = self._analysed
        if (center_ratio, window_size) != (vol["center"], vol["window"]):
            res = self._run(vol["first"], vol["last"], vol["ufov"], vol["cfov"], 1 - center_ratio, window_size)
        else:
            res = vol["result"]
        self.frame_result["center_fov"] = res.center_fov
        return _center_border_ratio(res.row)

    def _run(self, first: int, last: int, ufov_erode: float, cfov_erode: float, center_erode: float, window_size: int):
        b = determine_binning(float(self.stack.metadata.PixelSpacing[0]))
        a = self._volume
        rows, mean, cleaned, masks = nat.tu_uniformity(nat.Context.default(), a[None], len(a), first, last - first, b,
                                                       (ufov_erode, cfov_erode, center_erode), int(window_size), self.threshold)
        shape = (-(-a.shape[1] // b), -(-a.shape[2] // b))
        return TomographicUniformityVolume(rows[0], int(window_size), shape, _DeviceArrays(cleaned, masks, mean), 0)

    def analyze(self, first_frame: int = 0, last_frame: int = -1, ufov_ratio: float = 0.8, cfov_ratio: float = 0.75,
                center_ratio: float = 0.4, threshold: float = 0.75, window_size: int = 5) -> None:
        """Uniformity of the mean of slices `first_frame` up to (not including) `last_frame` (0-based; negative counts from the end),
        as PlanarUniformity.analyze with `ufov_ratio`, `cfov_ratio`, `threshold` and `window_size`, and the center-to-border ratio of
        a center FOV of `center_ratio` x `ufov_ratio`."""
        self.threshold = threshold
        first, last = _slab(len(self.stack.frames), first_frame, last_frame)
        frame0 = self.stack.frames[0]
        self.first_frame, self.last_frame = first + 1, last + 1
        if last == 0:                       # an empty slab: an all-nan mean frame with nothing above the threshold
            self.stack.frames = [frame0]
            frame0.array = np.full(np.shape(frame0.array), np.nan)
            _warn_empty_slab()
            raise ValueError(_EMPTY_MAX)
        if not hasattr(self, "_volume"):
            a = self.stack._pixels
            if a.dtype == np.uint8:
                a = a.astype(np.uint16)
            elif a.dtype != np.uint16:
                raise NotImplementedError(f"nuclear frames of dtype {a.dtype.name} are not supported (uint8 or uint16)")
            self._volume = a
        erode = (1 - ufov_ratio, 1 - cfov_ratio * ufov_ratio, 1 - center_ratio * ufov_ratio)
        res = self._run(first, last, *erode, window_size)
        self.stack.frames = [_SlabMeanFrame(frame0, res._arrays)]
        if res.status == nat.NM_NO_COMPONENT:
            if np.isnan(res.row["threshold"]):
                _warn_empty_threshold()
            raise ValueError(_EMPTY_MAX)
        self._analysed = {"first": first, "last": last, "ufov": erode[0], "cfov": erode[1], "center": center_ratio * ufov_ratio,
                          "window": window_size, "result": res}
        self.frame_results = {self.frame_key: {"ufov": res.ufov, "cfov": res.cfov, "binned_frame": res.binned_frame}}
        self.center_ratio = self.center_border_ratio(center_ratio=center_ratio * ufov_ratio, window_size=window_size)

    def results_data(self, as_dict: bool = False, as_json: bool = False, by_alias: bool = False, exclude: set[str] | None = None):
        """ResultsDataMixin's results_data: the reference's class resolves it before PlanarUniformity's"""
        return ResultsDataMixin.results_data(self, as_dict=as_dict, as_json=as_json, by_alias=by_alias, exclude=exclude)

    def _generate_results_data(self) -> TomographicUniformityResults:
        """Return the results as a structure."""
        return TomographicUniformityResults(
            cfov_integral_uniformity=self.frame_result["cfov"].integral_uniformity,
            cfov_differential_uniformity=self.frame_result["cfov"].differential_uniformity,
            ufov_integral_uniformity=self.frame_result["ufov"].integral_uniformity,
            ufov_differential_uniformity=self.frame_result["ufov"].differential_uniformity,
            center_border_ratio=self.center_ratio,
            first_frame=self.first_frame,
            last_frame=self.last_frame,
        )

    def results(self) -> str:
        """Return a string representation of the results."""
        return (
            f"Tomographic Uniformity results for {self.path.name}\n"
            f"Frames: {self.first_frame}:{self.last_frame}\n"
            f"CFOV Integral Uniformity: {self.frame_result['cfov'].integral_uniformity:.3f}%\n"
            f"CFOV Differential Uniformity: {self.frame_result['cfov'].differential_uniformity:.3f}%\n"
            f"UFOV Integral Uniformity: {self.frame_result['ufov'].integral_uniformity:.3f}%\n"
            f"UFOV Differential Uniformity: {self.frame_result['ufov'].differential_uniformity:.3f}%\n"
            f"Center-to-Border ratio: {self.center_ratio:.3f}\n"
        )


# ---------------------------------------------------------------------------------------------------- TomographicContrast
_EMPTY_MEAN = "Mean of empty slice"
_ALL_NAN_AXIS = "All-NaN axis encountered"
_BOUNDS_ORDER = "An upper bound is less than the corresponding lower bound."


def _michelson(array) -> float:
    """pylinac.core.contrast.michelson: (max - min) / (max + min), nan values ignored"""
    l_max, l_min = np.nanmax(array), np.nanmin(array)
    return (l_max - l_min) / (l_max + l_min)


def create_sphere_mask(array_shape: tuple[float, float, float], row: float, col: float, zed: float, radius: float) -> np.ndarray:
    """A mask of a sphere in an array (nuclear.py:1825-1835)."""
    z, y, x = np.ogrid[: array_shape[0], : array_shape[1], : array_shape[2]]
    return (x - col) ** 2 + (y - row) ** 2 + (z - zed) ** 2 <= radius**2


def sample_sphere(array: np.ndarray, row: float, col: float, zed: float, radius: float) -> np.ndarray:
    """A float64 copy of `array` that is nan outside the sphere (nuclear.py:1838-1847)."""
    sphere_mask = create_sphere_mask(array.shape, row=row, col=col, zed=zed, radius=radius)
    sphere_sample = np.full(array.shape, np.nan)
    sphere_sample[sphere_mask] = array[sphere_mask]
    return sphere_sample


def contrast_f(coords: np.ndarray, array: np.ndarray, radius: float, uniformity_baseline: float) -> float:
    """The objective of the sphere search (nuclear.py:1850-1856): -michelson([sphere mean, baseline]) x 100.  The device runs it
    on the sphere's bounding box; this host version is the reference's."""
    col, row, zed = coords
    sample = sample_sphere(array, col=col, row=row, zed=zed, radius=radius)
    return -_michelson(np.asarray([np.nanmean(sample), uniformity_baseline])) * 100


class TomographicROI:
    """One sphere at the searched position (nuclear.py:1553-1593).  The analysis gives its exact sum, count and min from the device;
    built by hand (without `stats`), it samples `array3d` as the reference does.  ``sphere_array`` is built on first access."""

    def __init__(self, array3d: np.ndarray | None, uniformity_baseline: float, x: float, y: float, z: float, radius: float,
                 number: str | int, stats: tuple[int, int, int] | None = None):
        self.array3d, self.uniformity_baseline = array3d, uniformity_baseline
        self.x, self.y, self.z, self.radius, self.number = x, y, z, radius, number
        self._stats = stats

    @cached_property
    def sphere_array(self) -> tuple[np.ndarray]:
        """(the volume as float64, nan outside the sphere,): a 1-tuple, as the reference builds it"""
        if self.array3d is None:
            raise RuntimeError("this ROI was analysed from a device batch and keeps no host volume")
        return (sample_sphere(self.array3d, col=self.x, row=self.y, zed=self.z, radius=self.radius),)

    @property
    def mean_value(self) -> float:
        if self._stats is None:
            return float(np.nanmean(self.sphere_array))
        s, n, _ = self._stats
        if n == 0:
            warnings.warn(_EMPTY_MEAN, RuntimeWarning, stacklevel=2)
            return math.nan
        return float(np.float64(s) / np.float64(n))

    @property
    def min_value(self) -> float:
        if self._stats is None:
            return float(np.nanmin(self.sphere_array))
        if self._stats[1] == 0:
            warnings.warn(_ALL_NAN_AXIS, RuntimeWarning, stacklevel=2)
            return math.nan
        return float(self._stats[2])

    @property
    def mean_contrast(self) -> float:
        return _michelson(np.asarray([self.mean_value, self.uniformity_baseline])) * 100

    @property
    def max_contrast(self) -> float:
        return _michelson(np.asarray([self.min_value, self.uniformity_baseline])) * 100


class TomgraphicSphere(TypedDict):
    x: float
    y: float
    z: float
    radius: float
    mean: float
    mean_contrast: float
    max_contrast: float


class TomographicContrastResults(ResultBase):
    uniformity_baseline: float  #:
    spheres: dict[str, TomgraphicSphere]  #:


def _slice_data(rows: np.ndarray) -> dict[str, dict]:
    """slice_data (nuclear.py:1620-1658) from the device rows of one volume's slices: the reference's dict, its warnings for slices
    with an empty FOV, and its area filter"""
    uniformities = {}
    for idx, r in enumerate(rows):
        if r["status"] == nat.NT_NO_COMPONENT:
            continue
        if r["area"] == 0:                    # michelson's nanmax and nanmin, then nanmean, of an all-nan FOV
            warnings.warn(_ALL_NAN, RuntimeWarning, stacklevel=3)
            warnings.warn(_ALL_NAN, RuntimeWarning, stacklevel=3)
            warnings.warn(_EMPTY_MEAN, RuntimeWarning, stacklevel=3)
        uniformities[str(idx + 1)] = {
            "fov diameter": int(r["longest"]) - int(r["erosion"]),
            "center": Point(x=np.float64(r["centroid_col"]), y=np.float64(r["centroid_row"])),
            "area": int(r["area"]),
            "uniformity": np.float64(r["uniformity"]),
            "value": np.float64(r["value"]),
        }
    median_area = np.median([v["area"] for v in uniformities.values()])
    std_area = np.std([v["area"] for v in uniformities.values()])
    return {k: v for k, v in uniformities.items() if v["area"] > median_area - std_area}


class TomographicContrastVolume:
    """The analysis of one volume of analyze_tomographic_contrast_batch: ``slice_rows`` (the device's NT_SLICE_DTYPE rows),
    ``slice_data``, ``uniformity_frame``, ``uniformity_value``, ``rois`` and ``searches`` (the NT_SPHERE_DTYPE rows).  A volume with
    no slice left keeps the reference's ValueError and raises it from ``raise_for_status()`` and every other attribute."""

    def __init__(self, slice_rows: np.ndarray, slice_data: dict):
        self.slice_rows, self.slice_data = slice_rows, slice_data
        self.error: Exception | None = None
        self.searches = np.zeros(0, nat.NT_SPHERE_DTYPE)
        self._rois: dict[str, TomographicROI] = {}

    def raise_for_status(self) -> None:
        if self.error is not None:
            raise self.error

    @property
    def uniformity_frame(self) -> str:
        """The frame with the most uniformity."""
        return min(self.slice_data, key=lambda x: self.slice_data.get(x)["uniformity"])

    @property
    def uniformity_value(self) -> float:
        return self.slice_data[self.uniformity_frame]["value"]

    @property
    def rois(self) -> dict[str, TomographicROI]:
        self.raise_for_status()
        return self._rois


def _sphere_inputs(out: list[TomographicContrastVolume], pixel_size_mm: float, sphere_diameters_mm, sphere_angles, search_window_px,
                   search_slices) -> tuple[np.ndarray, list[tuple[int, float]]]:
    """the host selection (nuclear.py:1693-1712): the NT_SPHERE_IN_DTYPE rows of every sphere search of the volumes of `out`, and
    each row's (volume, radius).  A volume with no slice left gets the reference's ValueError and no row."""
    if search_window_px < 0 or search_slices < 0:
        raise ValueError(_BOUNDS_ORDER)
    if search_window_px == 0 or search_slices == 0:
        raise NotImplementedError("a search window of zero fixes a variable, which scipy's minimize handles apart; not supported")
    spheres, owners = [], []
    for v, res in enumerate(out):
        data = res.slice_data
        if not data:
            res.error = ValueError(_EMPTY_MAX)
            continue
        start = max(data, key=lambda x: data[x]["uniformity"])    # the least uniform slice, usually near the spheres
        unif, unif_z = data[start], int(start) - 1
        baseline = res.uniformity_value
        for angle, diameter in zip(sphere_angles, sphere_diameters_mm):
            distance = math.sqrt(unif["area"] / math.pi) * 0.65
            radius = diameter / (2 * pixel_size_mm)
            col_x, row_y = direction_to_coords(unif["center"].x, unif["center"].y, distance, angle)
            spheres.append(((col_x, row_y, unif_z), (col_x - search_window_px, row_y - search_window_px, unif_z - search_slices),
                            (col_x + search_window_px, row_y + search_window_px, unif_z + search_slices), radius**2, baseline, v))
            owners.append((v, radius))
    inp = np.zeros(len(spheres), nat.NT_SPHERE_IN_DTYPE)
    for k, (x0, lb, ub, r2, baseline, v) in enumerate(spheres):
        inp[k] = (x0, lb, ub, r2, baseline, v, 0)
    return inp, owners


def _search_spheres(ctx, volumes, host, nz: int, out: list[TomographicContrastVolume], pixel_size_mm: float, sphere_diameters_mm,
                    sphere_angles, search_window_px, search_slices) -> None:
    """one device call for every sphere search of the volumes of `out`, and their ROIs"""
    inp, owners = _sphere_inputs(out, pixel_size_mm, sphere_diameters_mm, sphere_angles, search_window_px, search_slices)
    found = nat.nt_spheres(ctx, volumes, nz, inp, 600, 600)
    for k, ((v, radius), s) in enumerate(zip(owners, found)):
        res = out[v]
        res.searches = np.concatenate([res.searches, found[k:k + 1]])
        for _ in range(int(s["n_empty"])):
            warnings.warn(_EMPTY_MEAN, RuntimeWarning, stacklevel=2)
        col, row, zed = (np.float64(c) for c in s["x"])
        number = len(res._rois) + 1
        roi = TomographicROI(None if host is None else host[v], res.uniformity_value, col, row, zed, radius, number,
                             stats=(int(s["sum"]), int(s["count"]), int(s["min"])))
        roi._search = s                       # the device row: nfev, nit, status, n_empty, res.fun
        res._rois[str(number)] = roi


def analyze_tomographic_contrast_batch(volumes, pixel_size_mm: float, sphere_diameters_mm: Sequence[float] = (38, 31.8, 25.4, 19.1, 15.9, 12.7),
                                       sphere_angles: Sequence[float] = (-10, -70, -130, -190, 110, 50), ufov_ratio: float = 0.8,
                                       search_window_px: int = 5, search_slices: int = 3, *, slices_per_volume: int | None = None,
                                       device: int | None = None) -> list[TomographicContrastVolume]:
    """``TomographicContrast.analyze`` for every volume of `volumes`: a uint16 [n, z, h, w] (or [z, h, w]) ndarray, uint8 widened on
    the host, or a device Batch of n x z slices with ``slices_per_volume=z``.  One device call analyses every slice, the host selects
    the slices in the reference's own expressions, and one device call runs every sphere search.  Mismatched diameters and angles
    raise ValueError after the slice stage, as in the reference."""
    if isinstance(volumes, nat.Batch):
        (n, h, w), dt = volumes.shape_dtype
        if dt != np.uint16:
            raise NotImplementedError(f"nuclear frames of dtype {np.dtype(dt).name} are not supported (uint8 or uint16)")
        if slices_per_volume is None or slices_per_volume < 1 or n % slices_per_volume:
            raise ValueError(f"slices_per_volume must divide the batch's {n} slices, got {slices_per_volume}")
        nz, host = int(slices_per_volume), None
    else:
        a = np.asarray(volumes)
        if a.dtype == np.uint8:
            a = a.astype(np.uint16)
        elif a.dtype != np.uint16:
            raise NotImplementedError(f"nuclear frames of dtype {a.dtype.name} are not supported (uint8 or uint16)")
        if a.ndim not in (3, 4):
            raise ValueError(f"volumes must be [n, z, h, w] or [z, h, w], got {a.ndim}-D")
        host = a[None] if a.ndim == 3 else a
        nz = host.shape[1]
        volumes = host
    ctx = nat.Context.default(device)
    rows = nat.nt_slices(ctx, volumes, nz, 1 - ufov_ratio)
    out = [TomographicContrastVolume(r, _slice_data(r)) for r in rows.reshape(-1, nz)]
    if len(sphere_diameters_mm) != len(sphere_angles):
        raise ValueError("The number of sphere diameters and angles must be the same.")
    _search_spheres(ctx, volumes, host, nz, out, pixel_size_mm, sphere_diameters_mm, sphere_angles, search_window_px, search_slices)
    return out


@capture_warnings
class TomographicContrast(ResultsDataMixin[TomographicContrastResults]):
    """Sphere contrast of a reconstructed SPECT volume, such as a Jaszczak phantom (nuclear.py:1606-1822)."""

    rois: dict[str, TomographicROI]

    def __init__(self, path: str | Path):
        super().__init__()
        self.stack = NMImageStack(path)
        self.path = Path(path)

    @cached_property
    def slice_data(self) -> dict[str, dict[str, float | Point]]:
        """per kept slice (1-based key): its FOV diameter, center, area, uniformity and mean value"""
        if "ufov_ratio" in self.__dict__:
            return _slice_data(nat.nt_slices(nat.Context.default(), self._volume(), len(self.stack.frames), 1 - self.ufov_ratio))
        # before analyze(): the reference reads ufov_ratio at the first slice with a component, so a volume without one gives {}
        rows = nat.nt_slices(nat.Context.default(), self._volume(), len(self.stack.frames), 0.0)
        if np.any(rows["status"] == nat.NT_OK):
            return self.ufov_ratio
        return _slice_data(rows)

    def _volume(self) -> np.ndarray:
        a = self.stack._pixels
        if a.dtype == np.uint8:
            return a.astype(np.uint16)
        if a.dtype != np.uint16:
            raise NotImplementedError(f"nuclear frames of dtype {a.dtype.name} are not supported (uint8 or uint16)")
        return a

    @property
    def uniformity_frame(self) -> str:
        """The frame with the most uniformity."""
        return min(self.slice_data, key=lambda x: self.slice_data.get(x)["uniformity"])

    @property
    def uniformity_value(self) -> float:
        return self.slice_data[self.uniformity_frame]["value"]

    def analyze(self, sphere_diameters_mm: Sequence[float] = (38, 31.8, 25.4, 19.1, 15.9, 12.7),
                sphere_angles: Sequence[float] = (-10, -70, -130, -190, 110, 50), ufov_ratio: float = 0.8, search_window_px: int = 5,
                search_slices: int = 3) -> None:
        """Find each sphere (`sphere_diameters_mm`, at `sphere_angles` degrees) within `search_window_px` pixels and `search_slices`
        slices of its nominal position by a bounded Nelder-Mead search for the best contrast against the most uniform slice."""
        self.ufov_ratio = ufov_ratio
        data = self.slice_data
        if len(sphere_diameters_mm) != len(sphere_angles):
            raise ValueError("The number of sphere diameters and angles must be the same.")
        if not data:
            raise ValueError(_EMPTY_MAX)
        res = TomographicContrastVolume(None, data)
        volume = self._volume()
        _search_spheres(nat.Context.default(), volume, volume[None], len(volume), [res], float(self.stack.metadata.PixelSpacing[0]),
                        sphere_diameters_mm, sphere_angles, search_window_px, search_slices)
        self.rois = res.rois

    def results(self) -> str:
        """Return a string representation of the results."""
        s = f"Tomographic Contrast results for {self.path.name}\n"
        s += f"Uniformity baseline: {self.uniformity_value:.1f}\n"
        for idx, roi in self.rois.items():
            s += (f"Sphere {idx}: X={roi.x:.2f},Y={roi.y:.2f},Z={roi.z:.2f} Mean: {roi.mean_value:.2f}; "
                  f"Mean Contrast: {roi.mean_contrast:.2f}; Max Contrast: {roi.max_contrast:.2f}\n")
        return s

    def _generate_results_data(self) -> TomographicContrastResults:
        return TomographicContrastResults(
            uniformity_baseline=self.uniformity_value,
            spheres={idx: TomgraphicSphere(x=roi.x, y=roi.y, z=roi.z, radius=roi.radius, mean=roi.mean_value,
                                           mean_contrast=roi.mean_contrast, max_contrast=roi.max_contrast)
                     for idx, roi in self.rois.items()},
        )


# ---------------------------------------------------------------------------------------------------- QuadrantResolution
_QUADRANT_ANGLES = (45, -45, -135, 135)


def _four_bar_widths(bar_widths: Sequence[float]) -> np.ndarray:
    """the line pairs per mm of the four bar widths; any other number raises the reference's ValueError"""
    if len(bar_widths) != 4:
        raise ValueError("Must have 4 bar widths")
    return 1 / (2 * np.asarray(bar_widths))


def _quadrant_centers(rows: int, columns: int, bar_widths: Sequence[float], distance_from_center_mm: float) -> dict:
    """{bar width: ROI centre} in the reference's order and expressions: the phantom centre is Point(Rows / 2, Columns / 2), so the
    rows give x; a repeated bar width keeps its first position and its last centre.  Distances are used as pixels."""
    img_center = Point(rows / 2, columns / 2)
    centers = {}
    for angle, spacing in zip(_QUADRANT_ANGLES, bar_widths):
        centers[spacing] = HighContrastDiskROI._get_shifted_center(angle, distance_from_center_mm, img_center)
    return centers


class QuadrantResolutionFrame:
    """The analysis of one frame of analyze_quadrant_resolution_batch: the ROIs' statistics (lists in ROI order: ``counts``,
    ``means``, ``stds``, ``medians``, ``mins``, ``maxs``), their ``centers`` and ``bar_widths``, and the reference's ``mtf`` and
    ``quadrants``, which raise the reference's exceptions.  An empty ROI has a NaN mean, std and median, without numpy's warnings."""

    def __init__(self, lpmm: np.ndarray, centers: dict, stats: dict):
        self.lpmm, self.bar_widths, self.centers = lpmm, list(centers), list(centers.values())
        self.counts, self.means, self.stds = stats["count"], stats["mean"], stats["std"]
        self.medians, self.mins, self.maxs = stats["median"], stats["min"], stats["max"]

    @cached_property
    def mtf(self) -> MomentMTF:
        return MomentMTF(self.lpmm, self.means, self.stds)

    @property
    def quadrants(self) -> dict[str, dict[str, float]]:
        """QuadrantResolutionResults.quadrants"""
        return _quadrants(self.mtf)


def analyze_quadrant_resolution_batch(frames, bar_widths: Sequence[float], roi_diameter_mm: float = 70,
                                      distance_from_center_mm: float = 130, *, device: int | None = None) -> list[QuadrantResolutionFrame]:
    """``QuadrantResolution.analyze(bar_widths, roi_diameter_mm, distance_from_center_mm)`` for every frame of `frames` (an [n, h, w]
    or [h, w] ndarray or a device Batch, any dtype the disk statistics read), with the statistics of all its disks from one device
    call.  Each frame is analysed as QuadrantResolution analyses frame 0 of an h x w file.  The bar-width count and a disk beyond the
    frame raise the reference's ValueError and IndexError before any device call."""
    lpmm = _four_bar_widths(bar_widths)
    if isinstance(frames, nat.Batch):
        (n, h, w), _ = frames.shape_dtype
    else:
        frames = np.asarray(frames)
        frames = frames[None] if frames.ndim == 2 else frames
        if frames.ndim != 3:
            raise ValueError(f"frames must be [n, h, w] or [h, w], got {frames.ndim}-D")
        frames = disk_stats_dtype(frames)
        n, h, w = frames.shape
    centers = _quadrant_centers(h, w, bar_widths, distance_from_center_mm)
    for c in centers.values():
        check_disk_bounds((h, w), c.y, c.x, roi_diameter_mm)
    disks = [(f, c.y, c.x, roi_diameter_mm) for f in range(n) for c in centers.values()]
    out = nat.disk_stats(nat.Context.default(device), frames, disks)
    k = len(centers)
    return [QuadrantResolutionFrame(lpmm, centers, {name: [float(v) for v in a[f * k:(f + 1) * k]] for name, a in out.items()})
            for f in range(n)]


def _quadrants(mtf: MomentMTF) -> dict[str, dict[str, float]]:
    return {
        f"{idx + 1}": {"mtf": m, "fwhm": fwhm, "lpmm": lpmm, "spacing": 1 / (lpmm * 2)}
        for idx, ((lpmm, m), fwhm) in enumerate(zip(mtf.mtfs.items(), mtf.fwhms.values()))
    }


class QuadrantResolutionResults(ResultBase):
    quadrants: dict[str, dict[str, float]]  #: quadrant idx: {'mtf': mtf, 'fwhm': fwhm, 'lpmm': lpmm, 'spacing': bar width}


@capture_warnings
class QuadrantResolution(ResultsDataMixin[QuadrantResolutionResults]):
    """MTF and FWHM of a 4-quadrant bar phantom image (nuclear.py:1248-1367): the moments MTF of Hander et al. of one disk ROI per
    quadrant of frame 0."""

    rois: dict[float, HighContrastDiskROI]
    mtf: MomentMTF

    def __init__(self, path: str | Path) -> None:
        super().__init__()
        self.stack = NMImageStack(path)
        self.path = Path(path)

    def analyze(self, bar_widths: Sequence[float], roi_diameter_mm: float = 70, distance_from_center_mm: float = 130) -> None:
        """The MTF and FWHM of each quadrant, from disk ROIs of `roi_diameter_mm` (used as a radius in pixels) whose centres lie
        `distance_from_center_mm` (pixels) from the image centre.  `bar_widths`: the four bar widths in mm."""
        lpmm = _four_bar_widths(bar_widths)
        centers = _quadrant_centers(self.stack.metadata.Rows, self.stack.metadata.Columns, bar_widths, distance_from_center_mm)
        self.rois = {spacing: HighContrastDiskROI(self.stack.frames[0], radius=roi_diameter_mm, center=c, contrast_threshold=0)
                     for spacing, c in centers.items()}
        fill_disk_stats(list(self.rois.values()))
        self.mtf = MomentMTF.from_high_contrast_diskset(lpmm, list(self.rois.values()))

    def results(self) -> str:
        """Return a string representation of the results."""
        s = f"Quadrant Resolution results for {self.path.name}\n"
        for quadrant, ((lpmm, mtf), fwhm) in enumerate(zip(self.mtf.mtfs.items(), self.mtf.fwhms.values())):
            spacing = 1 / (lpmm * 2)
            s += f"Quadrant {quadrant + 1}; Bar width: {spacing:.2f}mm; FWHM: {fwhm:.3f}mm; MTF: {mtf:.3f}\n"
        return s

    def _generate_results_data(self) -> QuadrantResolutionResults:
        """Return the results as a structure."""
        return QuadrantResolutionResults(quadrants=_quadrants(self.mtf))
