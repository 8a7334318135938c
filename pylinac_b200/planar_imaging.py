"""Light / radiation field coincidence phantoms -- drop-in for the light/rad classes of ``pylinac.planar_imaging``
(planar_imaging.py:1169-1727): ``StandardImagingFC2`` and its subclasses ``IMTLRad``, ``DoselabRLf``, ``IsoAlign`` and ``SNCFSQA``,
with ``LightRadResult``.  ``pylinac_b200.contrib.quasar.QuasarLightRadScaling`` builds on them.

Same constructor (``filepath``, ``normalize=True``, ``image_kwargs``), ``analyze(invert, fwxm, bb_edge_threshold_mm,
kernel_size_multiplier)``, attributes (``field_center``, ``field_width_x`` / ``_y``, ``bb_center``, ``bb_centers``, ``epid_center``),
properties, ``results()`` and ``results_data()`` as the reference.  The pixel work -- ground / normalize, check_inversion, the strip
profiles and their FWXM edges, both 3 x 3 medians, the adaptive histogram equalisation of near-edge BBs and every BB search -- is one
device call per batch (``epid_lightrad_analyze``, csrc/lightrad.cu); ``analyze_batch(frames, dpmm, phantom=...)`` runs n frames at
once and the classes go through it with n = 1.  The loaded ``image`` keeps its pixels: the device applies ground / normalize /
invert as a map of the integer frame.  Not here: plotting, ``publish_pdf``, QuAAC export, ``from_demo_image`` / ``from_url``, and
the image-quality phantoms.
"""
from __future__ import annotations

from collections.abc import Sequence

import numpy as np
from pydantic import Field

from . import _native as nat
from .core import image
from .core.geometry import Point, Vector
from .core.utilities import ResultBase, ResultsDataMixin
from .core.warnings import capture_warnings


def percent_integral_uniformity(max: float, min: float) -> float:
    """planar_imaging.py:140-143: 100 * (1 - (max - min + 1e-6) / (max + min + 1e-6)); the constant keeps a blank disk finite."""
    return 100 * (1 - (max - min + 1e-6) / (max + min + 1e-6))


class LightRadResult(ResultBase):
    """planar_imaging.py:1169-1198"""

    field_size_x_mm: float = Field(description="The size of the field in the x-direction/crossplane in mm.", title="Field Size X (mm)")
    field_size_y_mm: float = Field(description="The size of the field in the y-direction/inplane in mm.", title="Field Size Y (mm)")
    field_epid_offset_x_mm: float = Field(description="The offset of the field center from the EPID/image center in the x-direction/crossplane in mm.",
                                          title="Field->EPID X offset (mm)")
    field_epid_offset_y_mm: float = Field(description="The offset of the field center from the EPID/image center in the y-direction/inplane in mm.",
                                          title="Field->EPID Y offset (mm)")
    field_bb_offset_x_mm: float = Field(description="The offset of the field center from the BB center in the x-direction/crossplane in mm.",
                                        title="Field->BB X offset (mm)")
    field_bb_offset_y_mm: float = Field(description="The offset of the field center from the BB center in the y-direction/inplane in mm.",
                                        title="Field->BB Y offset (mm)")


_SET_FIXED, _SET_FC2, _SET_QUASAR = 0, 1, 2
_STATUS_OK, _STATUS_NO_FIELD, _STATUS_MISMATCH, _STATUS_NO_BB, _STATUS_CAPACITY = 0, 1, 2, 3, 4


def _params(phantom, dpmm: float, normalize: bool, invert: bool, fwxm: float, bb_edge_threshold_mm: float,
            kernel_size_multiplier: float) -> nat.LrParams:
    bb_set, mode = phantom._device_bb_set()
    p = nat.LrParams()
    p.dpmm = float(dpmm)
    p.fwxm = float(fwxm)
    p.bb_edge_threshold_mm = float(bb_edge_threshold_mm)
    p.bb_size_mm = float(phantom.bb_size_mm)
    p.bb_box_mm = float(phantom.bb_sampling_box_size_mm)
    p.strip_width_mm = float(phantom.field_strip_width_mm)
    p.quasar_offset_mm = float(getattr(phantom, "light_rad_bb_offset_mm", 0.0))
    p.set_mode = mode
    p.nbb = len(bb_set)
    for k, (x, y) in enumerate(bb_set.values()):
        p.bb_mm[2 * k], p.bb_mm[2 * k + 1] = float(x), float(y)
    if mode == _SET_FC2:
        for k, (x, y) in enumerate(phantom.bb_positions_15x15.values()):
            p.bb15_mm[2 * k], p.bb15_mm[2 * k + 1] = float(x), float(y)
    p.normalize = int(bool(normalize))
    p.invert = int(bool(invert))
    # _detect_bb_centers: kernel_size=int(round(bb_radius_px * kernel_size_multiplier)) (:1444-1449)
    p.clahe_kernel = int(round(phantom.bb_size_mm / 2 * dpmm * kernel_size_multiplier))
    p.scaling = int(getattr(phantom, "_scaling_search", False))
    return p


class LightRadFrame:
    """One frame's results (a row of the struct-of-arrays the device returns), materialised lazily."""

    def __init__(self, row, phantom, dpmm: float, shape):
        self.r = row
        self.phantom = phantom
        self.dpmm = dpmm
        self.shape = shape

    @property
    def status(self) -> int:
        return int(self.r["status"])

    @property
    def inverted(self) -> bool:
        """check_inversion() fired (before the ``invert`` argument)"""
        return bool(self.r["inverted"])

    @property
    def near_edge(self) -> list[bool]:
        """per BB: located on the adaptively equalised image"""
        return [bool(int(self.r["near_edge_mask"]) >> k & 1) for k in range(len(self._keys()))]

    def raise_for_status(self):
        s = self.status
        if s == _STATUS_NO_FIELD:
            raise IndexError("index 0 is out of bounds for axis 0 with size 0")      # peak_props["left_ips"][0] of no peak
        if s == _STATUS_MISMATCH:
            raise ValueError("The detected y and x field sizes were too different from one another. They should be within 1cm from each "
                             f"other. Detected field sizes: x={self.field_width_x:.2f}mm, y={self.field_width_y:.2f}mm")
        if s == _STATUS_NO_BB:
            need = 1 if int(self.r["failed_bb"]) < len(self._keys()) else nat.LR_SCALING
            raise ValueError(f"Couldn't find the minimum number of disks in the image. Found {int(self.r['n_found'])}; required: {need}")
        if s == _STATUS_CAPACITY:
            raise MemoryError("light/rad: a search window or candidate region exceeds the locator's device tile (EPID_LR_CAPACITY)")

    def _keys(self) -> list[str]:
        if self.phantom._device_bb_set()[1] == _SET_FC2 and int(self.r["large_set"]):
            return list(self.phantom.bb_positions_15x15)
        return list(self.phantom._device_bb_set()[0])

    @property
    def field_center(self) -> Point:
        return Point(float(self.r["field_center_x"]), float(self.r["field_center_y"]))

    @property
    def field_width_x(self) -> float:
        return float(self.r["field_width_x_mm"])

    @property
    def field_width_y(self) -> float:
        return float(self.r["field_width_y_mm"])

    @property
    def epid_center(self) -> Point:
        """image.center (core/image.py:526-533)"""
        return Point(self.shape[1] / 2 - 0.5, self.shape[0] / 2 - 0.5)

    @property
    def bb_centers(self) -> dict[str, Point]:
        self.raise_for_status()
        out = {k: Point(float(self.r["bb_x"][i]), float(self.r["bb_y"][i])) for i, k in enumerate(self._keys())}
        if self.phantom._virtual_center:
            # SNCFSQA._find_overall_bb_centroid (:1714-1727): the phantom centre is 4 cm from the TR marker
            out["Virtual Center"] = out["TR"] - Point(40 * self.dpmm, -40 * self.dpmm)
        return out

    @property
    def bb_center(self) -> Point:
        centers = self.bb_centers
        if self.phantom._virtual_center:
            return centers["Virtual Center"]
        return Point(x=np.mean([p.x for p in centers.values()]), y=np.mean([p.y for p in centers.values()]))

    @property
    def scaling_centers(self) -> list[Point]:
        self.raise_for_status()
        return [Point(float(self.r["scaling_x"][j]), float(self.r["scaling_y"][j])) for j in range(int(self.r["n_scaling"]))]

    @property
    def field_epid_offset_mm(self) -> Vector:
        e, f = self.epid_center, self.field_center
        return Vector(e.x - f.x, e.y - f.y) / self.dpmm

    @property
    def field_bb_offset_mm(self) -> Point:
        return (self.bb_center - self.field_center) / self.dpmm


class LightRadBatchResult(Sequence):
    def __init__(self, rows: np.ndarray, phantom, dpmm: float, shape):
        self.rows = rows
        self.phantom = phantom
        self.dpmm = dpmm
        self.shape = shape

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, i) -> LightRadFrame:
        return LightRadFrame(self.rows[i], self.phantom, self.dpmm, self.shape)


def analyze_batch(frames, dpmm: float, phantom=None, *, normalize: bool = True, device: int | None = None, invert: bool = False,
                  fwxm: int = 50, bb_edge_threshold_mm: float = 10, kernel_size_multiplier: float = 2.0) -> LightRadBatchResult:
    """``phantom(frame, normalize).analyze(invert, fwxm, bb_edge_threshold_mm, kernel_size_multiplier)`` for every frame of ``frames``
    (uint16 [n, h, w] ndarray or device Batch) in one device call.  ``phantom`` is one of the light/rad classes (default
    StandardImagingFC2); the rows are materialised per access and raise the reference's exceptions from ``raise_for_status()`` and
    the point attributes."""
    phantom = StandardImagingFC2 if phantom is None else phantom
    ctx = nat.Context.default(device)
    if isinstance(frames, nat.Batch):
        (_, h, w), _ = frames.shape_dtype
    else:
        a = np.asarray(frames)
        if a.dtype != np.uint16:
            raise TypeError("light/rad frames must be uint16")
        frames = a[None] if a.ndim == 2 else a
        h, w = frames.shape[1:]
    p = _params(phantom, dpmm, normalize, invert, fwxm, bb_edge_threshold_mm, kernel_size_multiplier)
    rows = nat.lightrad_analyze(ctx, frames, p)
    return LightRadBatchResult(rows, phantom, float(dpmm), (h, w))


@capture_warnings
class StandardImagingFC2(ResultsDataMixin[LightRadResult]):
    """planar_imaging.py:1240-1623"""

    common_name = "SI FC-2"
    bb_positions_10x10 = {"TL": [-40, -40], "BL": [-40, 40], "TR": [40, -40], "BR": [40, 40]}
    bb_positions_15x15 = {"TL": [-65, -65], "BL": [-65, 65], "TR": [65, -65], "BR": [65, 65]}
    bb_sampling_box_size_mm = 10
    field_strip_width_mm = 5
    bb_size_mm = 4
    bb_edge_threshold_mm: float
    kernel_size_multiplier: float
    bb_centers: dict[str, Point]
    _virtual_center = False

    def __init__(self, filepath, normalize: bool = True, image_kwargs: dict | None = None):
        super().__init__()
        self.image = image.load(filepath, **(image_kwargs or {}))
        self._normalize = normalize

    @classmethod
    def _device_bb_set(cls) -> tuple[dict, int]:
        """the nominal BB positions the device chooses from, and how it chooses (_determine_bb_set)"""
        return cls.bb_positions_10x10, _SET_FC2

    def analyze(self, invert: bool = False, fwxm: int = 50, bb_edge_threshold_mm: float = 10, kernel_size_multiplier: float = 2.0) -> None:
        """planar_imaging.py:1282-1305"""
        if self.image.dpmm is None:
            raise ValueError("The image has no dpmm; pass image_kwargs={'dpi': ...} for array input")
        self.bb_edge_threshold_mm = bb_edge_threshold_mm
        self.kernel_size_multiplier = kernel_size_multiplier
        frame = image.frame_u16(self.image, "light/rad")
        res = analyze_batch(frame[None], self.image.dpmm, type(self), normalize=self._normalize, invert=invert, fwxm=fwxm,
                            bb_edge_threshold_mm=bb_edge_threshold_mm, kernel_size_multiplier=kernel_size_multiplier)[0]
        self._frame = res
        if res.status == _STATUS_NO_FIELD:
            res.raise_for_status()
        self.field_center, self.field_width_x, self.field_width_y = res.field_center, res.field_width_x, res.field_width_y
        res.raise_for_status()
        self.bb_centers = res.bb_centers
        self.bb_center = res.bb_center
        self.epid_center = res.epid_center

    def results(self, as_list: bool = False) -> str | list[str]:
        """planar_imaging.py:1307-1323"""
        text = [
            f"{self.common_name} results:",
            f"File: {getattr(self.image, 'path', '')}",
            f"The detected inplane field size was {self.field_width_y:2.1f}mm",
            f"The detected crossplane field size was {self.field_width_x:2.1f}mm",
            f"The inplane field was {self.field_epid_offset_mm.y:2.1f}mm from the EPID CAX",
            f"The crossplane field was {self.field_epid_offset_mm.x:2.1f}mm from the EPID CAX",
            f"The inplane field was {self.field_bb_offset_mm.y:2.1f}mm from the BB inplane center",
            f"The crossplane field was {self.field_bb_offset_mm.x:2.1f}mm from the BB crossplane center",
        ]
        return text if as_list else "\n".join(text)

    @property
    def field_epid_offset_mm(self) -> Vector:
        """Field offset from CAX using vector difference"""
        e, f = self.epid_center, self.field_center
        return Vector(e.x - f.x, e.y - f.y) / self.image.dpmm

    @property
    def field_bb_offset_mm(self) -> Point:
        """Field offset from BB centroid using vector difference"""
        return (self.bb_center - self.field_center) / self.image.dpmm

    def _generate_results_data(self) -> LightRadResult:
        return LightRadResult(field_size_x_mm=self.field_width_x, field_size_y_mm=self.field_width_y,
                              field_epid_offset_x_mm=self.field_epid_offset_mm.x, field_epid_offset_y_mm=self.field_epid_offset_mm.y,
                              field_bb_offset_x_mm=self.field_bb_offset_mm.x, field_bb_offset_y_mm=self.field_bb_offset_mm.y)

    def _is_bb_near_edge(self, bb_position) -> bool:
        """planar_imaging.py:1614-1623 (the device takes the same decision per BB)"""
        threshold = self.bb_edge_threshold_mm
        return abs(bb_position[0]) > self.field_width_x / 2 - threshold or abs(bb_position[1]) > self.field_width_y / 2 - threshold


@capture_warnings
class IMTLRad(StandardImagingFC2):
    """The IMT light/rad phantom (planar_imaging.py:1626-1639)"""

    common_name = "IMT L-Rad"
    center_only_bb = {"Center": [0, 0]}
    bb_sampling_box_size_mm = 12
    field_strip_width_mm = 5
    bb_size_mm = 3

    @classmethod
    def _device_bb_set(cls):
        return cls.center_only_bb, _SET_FIXED


@capture_warnings
class DoselabRLf(StandardImagingFC2):
    """The Doselab light/rad phantom (planar_imaging.py:1642-1670)"""

    common_name = "Doselab RLf"
    bb_positions_10x10 = {"TL": [-17, -45], "BL": [-45, 17], "TR": [45, -17], "BR": [17, 45]}

    @classmethod
    def _device_bb_set(cls):
        return cls.bb_positions_10x10, _SET_FIXED


@capture_warnings
class IsoAlign(StandardImagingFC2):
    """The PTW Iso-Align light/rad phantom (planar_imaging.py:1673-1697)"""

    common_name = "PTW Iso-Align"
    bb_positions = {"Center": [0, 0], "Top": [0, -25], "Bottom": [0, 25], "Left": [-25, 0], "Right": [25, 0]}
    field_strip_width_mm = 10

    @classmethod
    def _device_bb_set(cls):
        return cls.bb_positions, _SET_FIXED


@capture_warnings
class SNCFSQA(StandardImagingFC2):
    """SNC FSQA light/rad phantom (planar_imaging.py:1700-1727): the offset marker at the top right is located and the phantom centre
    is the 'virtual centre' 4 cm from it in each direction."""

    common_name = "SNC FSQA"
    center_only_bb = {"TR": [40, -40]}
    field_strip_width_mm = 5
    _virtual_center = True

    @classmethod
    def _device_bb_set(cls):
        return cls.center_only_bb, _SET_FIXED
