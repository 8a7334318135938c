"""pylinac.nuclear (nuclear.py:39-500): MaxCountRate and PlanarUniformity of gamma-camera NM files.

PlanarUniformity's whole frame pipeline (binning, the NEMA 9-point filter, the threshold, the stray-pixel clean-up, the largest
component, both FOV erosions, integral and differential uniformity) runs in one device call per batch (csrc/nuclear.cu), bit-identical
to the reference.  The cleaned frames and FOV masks stay on the device until an attribute needs them.  MaxCountRate takes its exact
frame sums from epid_frame_stats.  The other nuclear tests are not ported yet (DESIGN.md section 6).
"""
from __future__ import annotations

import json
from collections.abc import Sequence
from pathlib import Path

import numpy as np
from pydantic import BaseModel

from . import _native as nat
from .core.image import NMImageStack
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

    def __init__(self, cleaned: nat.Batch | None, masks: nat.Batch | None):
        self._batches = {"cleaned": cleaned, "masks": masks}
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

    def __init__(self, name: str, window_size: int, row, k: int, shape: tuple[int, int], arrays: _DeviceArrays, frame: int):
        self.name = name
        self.window_size = window_size
        self._row, self._k, self._shape, self._arrays, self._frame = row, k, shape, arrays, frame

    @property
    def mask(self) -> np.ndarray:
        """the eroded binary of the frame (bool)"""
        return self._arrays.get("masks")[2 * self._frame + self._k].astype(bool)

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
