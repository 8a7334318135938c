"""VMAT QA (DRGS / DRMLC / DRCS) -- drop-in for the analysis path of ``pylinac.vmat`` (reference file cited per item).

``DRGS(image_paths=(a, b)).analyze(...)`` / ``DRMLC`` / ``DRCS`` keep the reference's signatures, attributes (``segments``,
``open_image``, ``dmlc_image``, ``ratio_image``, ``r_devs``, ``passed`` ...) and ``results_data()``.  Underneath:

* DRGS / DRMLC: the whole per-pair pipeline -- ground / corner inversion check of both images, the column-mean FWXM profiles that
  identify the open image and give the field centre, the per-segment mean / std of DMLC / open, R_dev -- is four CUDA launches
  (``epid_vmat_analyze``, csrc/vmat.cu); ``analyze_batch(images1, images2, dpmm, ...)`` runs n pairs at once.
* DRCS: image identification by the 10 x 10 median (device filter), ratio image (``epid_divide``), rotated segment statistics
  (``epid_roi_stats``) and the collimator spokes from two ``CircleProfile`` rings (``epid_circle_profile`` + ``epid_find_peaks``).

Not here: plotting, PDF, QuAAC export, ``from_url`` / ``from_demo_images`` (no network), ``from_zip``.
"""
from __future__ import annotations

import enum
import math
import warnings
from collections.abc import Sequence
from dataclasses import dataclass

import numpy as np
from pydantic import BaseModel, ConfigDict, Field

from . import _native as nat
from .core import image
from .core.geometry import Point
from .core.image import frame_u16
from .core.profile import CircleProfile, FWXMProfile, Normalization
from .core.roi import RectangleROI
from .core.utilities import ResultBase, ResultsDataMixin
from .core.warnings import capture_warnings


def wrap180(value):
    """core/scale.py:23-30"""
    return (value + 180) % 360 - 180


class ImageType(enum.Enum):
    """vmat.py:54-59"""

    DMLC = "dmlc"
    OPEN = "open"
    PROFILE = "profile"


class SegmentResult(BaseModel):
    """vmat.py:62-85"""

    model_config = ConfigDict(arbitrary_types_allowed=True)
    passed: bool = Field(description="A boolean indicating if the segment passed or failed.")
    x_position_mm: float = Field(description="The position of the segment ROI in mm from CAX (lateral offset if DRGS/DRMLC, radial distance if DRCS).")
    angular_position_deg: float = Field(description="The angle of the segment ROI in degrees.")
    r_corr: float = Field(description="R corrected (ratio)", title="R corrected (ratio)")
    r_dev: float = Field(description="R deviation (%)", title="R deviation (%)")
    center_x_y: tuple[float, float] = Field(description="The center of the segment in pixel coordinates.")
    stdev: float = Field(description="The standard deviation of the segment of the ratioed images (DMLC / Open)")


class CollimatorResult(BaseModel):
    """vmat.py:88-98"""

    model_config = ConfigDict(arbitrary_types_allowed=True)
    angle_deviation: float = Field(description="Collimator Deviation at angle")
    angle_nominal: float = Field(description="The nominal angle of the collimator", title="Nominal Angle (deg)")


class VMATResult(ResultBase):
    """vmat.py:101-128"""

    test_type: str = Field(description="The type of test that was performed as a string.")
    tolerance_percent: float = Field(description=" The tolerance used to determine if the test passed or failed.")
    max_deviation_percent: float = Field(description="The maximum deviation of any segment.", title="Max Deviation (%)")
    abs_mean_deviation: float = Field(description="The average absolute deviation of all segments.", title="Absolute Mean Deviation (%)")
    passed: bool = Field(description="A boolean indicating if the test passed or failed.")
    segment_data: list[SegmentResult] = Field(description="List of individual segment data.")
    named_segment_data: dict[str, SegmentResult] = Field(description="Named individual segment data.")


class DRCSResult(VMATResult):
    """vmat.py:131-139"""

    rotation_offset_deg: float = Field(description="The signed mean of the collimator angle deviations.", title="Rotation Offset (deg)")
    collimator_data: dict[str, CollimatorResult] = Field(description="List of individual collimator deviation data")


class Segment:
    """vmat.py:142-188.  The statistics are device reductions: DRGS / DRMLC segments carry the values ``epid_vmat_analyze`` computed
    for them (``RectangleROI`` geometry for the accessors); DRCS segments are ``RectangleROI`` reductions on the ratio image."""

    def __init__(self, center_point: Point, width: float, height: float, tolerance: float, rotation: float = 0.0, *, r_corr=None,
                 stdev=None, ratio_image=None):
        self.center = Point(center_point)
        self.width = width
        self.height = height
        self.rotation = rotation
        self.r_dev: float = 0.0
        self._tolerance = tolerance
        self._r_corr = r_corr
        self._stdev = stdev
        self._ratio_image = ratio_image
        if r_corr is None:
            roi = RectangleROI(ratio_image, width, height, self.center, rotation)
            st = roi._compute()
            self._r_corr = st["mean"] * 100
            self._stdev = st["std"]

    @property
    def r_corr(self) -> float:
        return float(self._r_corr)

    @property
    def stdev(self) -> float:
        return float(self._stdev)

    @property
    def passed(self) -> bool:
        return bool(abs(self.r_dev) < self._tolerance * 100)

    def get_bg_color(self) -> str:
        return "blue" if self.passed else "red"


@dataclass
class CollimatorDeviation:
    """vmat.py:191-223"""

    name: str
    angle_nominal: float
    points: tuple

    @staticmethod
    def calculate_angle_measured(point1: Point, point2: Point) -> float:
        dy = point2.y - point1.y
        dx = point2.x - point1.x
        angle_im = np.arctan2(dy, dx)
        return float(-(np.rad2deg(angle_im) + 90) % 360)

    @property
    def angle_measured(self) -> float:
        return self.calculate_angle_measured(self.points[0], self.points[1])

    @property
    def angle_deviation(self) -> float:
        return wrap180(self.angle_measured - self.angle_nominal)


def _make_params(dpmm, tolerance, segment_size_mm, offsets_mm, ground, check_inversion, invert_image_order) -> nat.VmatParams:
    if len(offsets_mm) > nat.VMAT_MAX_SEG:
        raise ValueError(f"at most {nat.VMAT_MAX_SEG} segments are supported, got {len(offsets_mm)}")
    p = nat.VmatParams()
    p.ground = int(bool(ground))
    p.check_inversion = int(bool(check_inversion))
    p.invert_image_order = int(bool(invert_image_order))
    p.nseg = len(offsets_mm)
    p.dpmm = float(dpmm)
    p.tolerance_percent = float(tolerance)
    p.seg_w_mm, p.seg_h_mm = float(segment_size_mm[0]), float(segment_size_mm[1])
    for i, o in enumerate(offsets_mm):
        p.offset_mm[i] = float(o)
    return p


class VMATBatchRow:
    """One pair of a batched run: the result row of ``epid_vmat_analyze`` with the reference's accessor names."""

    def __init__(self, row, nseg):
        self.r = row
        self.nseg = nseg

    def raise_for_status(self):
        if int(self.r["status"]) != 0:
            raise IndexError("a column-mean profile of the pair has no peak (the reference fails in FWXMProfile.field_edge_idx)")

    @property
    def open_is_first(self) -> bool:
        return bool(self.r["open_is_first"])

    @property
    def r_corrs(self) -> np.ndarray:
        return self.r["r_corr"][: self.nseg]

    @property
    def r_devs(self) -> np.ndarray:
        return self.r["r_dev"][: self.nseg]

    @property
    def stdevs(self) -> np.ndarray:
        return self.r["stdev"][: self.nseg]

    @property
    def passed(self) -> bool:
        return bool(self.r["passed"])

    @property
    def max_r_deviation(self) -> float:
        return float(self.r["max_r_deviation"])

    @property
    def avg_abs_r_deviation(self) -> float:
        return float(self.r["avg_abs_r_deviation"])

    @property
    def avg_r_deviation(self) -> float:
        return float(self.r["avg_r_deviation"])


def analyze_batch(images1, images2, dpmm: float, *, test: str = "DRGS", tolerance: float = 1.5, segment_size_mm=None, roi_config=None,
                  ground: bool = True, check_inversion: bool = True, invert_image_order: bool = False, device: int | None = None):
    """n (image 1, image 2) pairs [n, H, W] uint16 (either order: the open image is identified per pair) through the DRGS / DRMLC
    analysis on the GPU -> list of :class:`VMATBatchRow`."""
    cls = {"DRGS": DRGS, "DRMLC": DRMLC}[test.upper()]
    roi_config = roi_config or cls._default_roi_config()
    segment_size_mm = segment_size_mm or (5, 100)
    offsets = [v["offset_mm"] for v in roi_config.values()]
    p = _make_params(dpmm, tolerance, segment_size_mm, offsets, ground, check_inversion, invert_image_order)
    rows = nat.vmat_analyze(nat.Context.default(device), images1, images2, p)
    return [VMATBatchRow(rows[i], len(offsets)) for i in range(len(rows))]


class VMATBase(ResultsDataMixin[VMATResult]):
    """vmat.py:226-725"""

    _result_header: str = ""
    _result_short_header: str = ""
    text_rotation = 0

    @classmethod
    def from_zip(cls, path, **kwargs):
        """vmat.py:288-301: both images from a ZIP archive."""
        with image.TemporaryZipDirectory(path) as tmp:
            return cls(image_paths=image.retrieve_image_files(tmp), **kwargs)

    def __init__(self, image_paths: Sequence, ground=True, check_inversion=True, **kwargs):
        super().__init__()
        ground = kwargs.pop("ground", False) or ground
        check_inversion = kwargs.pop("check_inversion", False) or check_inversion
        if len(image_paths) != 2:
            raise ValueError("Exactly 2 images (open, DMLC) must be passed")
        self._ground, self._check_inversion = bool(ground), bool(check_inversion)
        image1, image2 = image.load(image_paths[0], **kwargs), image.load(image_paths[1], **kwargs)
        # the integer frames the device path analyses (taken before the image objects are grounded / inverted)
        self._raw = [self._frame(image1), self._frame(image2)]
        for img in (image1, image2):      # _load_images / _check_inversion (vmat.py:348-357, 721-725): device operators of BaseImage
            if ground:
                img.ground()
            if check_inversion:
                img.check_inversion()
        self._images = [image1, image2]
        self._identify_images(image1, image2)
        self.segments: list[Segment] = []
        self._tolerance = 0

    def _frame(self, img) -> np.ndarray:
        if not self._ground and getattr(img, "_stored", None) is not None and getattr(img, "_stored_map", (1.0, 0.0, False))[:2] != (1.0, 0.0):
            raise ValueError("ground=False on a rescaled DICOM image: the ratio depends on the rescale intercept; use ground=True")
        return np.ascontiguousarray(frame_u16(img, "VMAT"))

    @property
    def passed(self) -> bool:
        return all(segment.passed for segment in self.segments)

    @property
    def r_devs(self) -> np.ndarray:
        return np.array([segment.r_dev for segment in self.segments])

    @property
    def avg_abs_r_deviation(self) -> float:
        return float(np.abs(self.r_devs).mean())

    @property
    def avg_r_deviation(self) -> float:
        return float(self.r_devs.mean())

    @property
    def max_r_deviation(self) -> float:
        return float(np.max(np.abs(self.r_devs)))

    @property
    def ratio_image(self) -> np.ndarray:
        """``dmlc_image.array / open_image.array`` (vmat.py:339), computed on the device on first access."""
        if getattr(self, "_ratio", None) is None:
            self._ratio = nat.divide(nat.Context.default(), np.asarray(self.dmlc_image.array), np.asarray(self.open_image.array))
        return self._ratio

    def _update_r_corrs(self):
        """vmat.py:408-412"""
        avg_r_corr = np.array([segment.r_corr for segment in self.segments]).mean()
        for segment in self.segments:
            segment.r_dev = ((segment.r_corr / avg_r_corr) * 100) - 100

    def results(self) -> str:
        """vmat.py:368-384"""
        passfail_str = "PASS" if self.passed else "FAIL"
        string = f"{self._result_header}\nTest Results (Tol. +/-{self._tolerance * 100:2.2}%): {passfail_str}\n"
        string += f"Max Deviation: {self.max_r_deviation:2.3}%\nAbsolute Mean Deviation: {self.avg_abs_r_deviation:2.3}%"
        return string


class VMATLinearBase(VMATBase):
    """vmat.py:727-841: DRGS / DRMLC.  Everything numerical is ``epid_vmat_analyze``."""

    text_rotation = 90

    @property
    def default_segment_size_mm(self) -> tuple[float, float]:
        return 5, 100

    @classmethod
    def _default_roi_config(cls) -> dict:
        raise NotImplementedError

    @property
    def default_roi_config(self) -> dict:
        return self._default_roi_config()

    def _run(self, tolerance, segment_size_mm, roi_config, invert_image_order):
        offsets = [v["offset_mm"] for v in roi_config.values()]
        dpmm = self._images[0].dpmm
        p = _make_params(dpmm, tolerance, segment_size_mm, offsets, self._ground, self._check_inversion, invert_image_order)
        row = nat.vmat_analyze(nat.Context.default(), self._raw[0], self._raw[1], p)[0]
        VMATBatchRow(row, len(offsets)).raise_for_status()
        return row

    def _identify_images(self, image1, image2):
        """vmat.py:739-764 (the decision is taken on the device from the two column-mean profiles)"""
        row = self._run(1.5, self.default_segment_size_mm, self.default_roi_config, False)
        first_open = bool(row["open_is_first"])
        self.open_image, self.dmlc_image = (image1, image2) if first_open else (image2, image1)
        self._swapped = False

    def _roi_profiles(self, image1, image2) -> list[FWXMProfile]:
        """vmat.py:766-783 (qualitative profiles for display; the analysis itself uses the device copies)"""
        profiles = []
        for orig in (image1, image2):
            a = np.asarray(orig.array)
            img = image.ArrayImage(a.copy())
            img.ground()
            img.check_inversion()
            profile = FWXMProfile(np.mean(img.array, axis=0), ground=True, normalization=Normalization.BEAM_CENTER)
            profile.stretch()
            profile.normalize(np.percentile(profile.values, 90))
            profiles.append(profile)
        return profiles

    def analyze(self, tolerance: float | int = 1.5, segment_size_mm: tuple | None = None, roi_config: dict | None = None,
                invert_image_order: bool = False):
        """vmat.py:309-346"""
        if segment_size_mm is None:
            segment_size_mm = self.default_segment_size_mm
        if roi_config is None:
            roi_config = self.default_roi_config
        # the swap acts on whatever the previous calls left behind, like the reference (two inverting calls swap back)
        if invert_image_order:
            self.open_image, self.dmlc_image = self.dmlc_image, self.open_image
            self._swapped = not self._swapped
        self._tolerance = tolerance / 100
        self.roi_config = roi_config
        self._ratio = None
        row = self._run(tolerance, segment_size_mm, roi_config, self._swapped)
        if int(row["center_warning"]):
            warnings.warn("The detected VMAT field center is outside the center third of the image; using the image center instead.",
                          UserWarning)
        dpmm = self.open_image.dpmm
        self.segments = []
        for i in range(len(roi_config)):
            seg = Segment(Point(float(row["center_x"][i]), float(row["center_y"][i])), width=segment_size_mm[0] * dpmm,
                          height=segment_size_mm[1] * dpmm, tolerance=self._tolerance, r_corr=float(row["r_corr"][i]),
                          stdev=float(row["stdev"][i]))
            seg.r_dev = float(row["r_dev"][i])
            self.segments.append(seg)
        self._row = row

    def _generate_results_data(self) -> VMATResult:
        """vmat.py:785-812"""
        segment_data, named = [], {}
        for segment, (roi_name, roi_data) in zip(self.segments, self.roi_config.items()):
            sr = SegmentResult(passed=segment.passed, r_corr=segment.r_corr, r_dev=segment.r_dev, center_x_y=(segment.center.x, segment.center.y),
                               x_position_mm=roi_data["offset_mm"], stdev=segment.stdev, angular_position_deg=0)
            segment_data.append(sr)
            named[roi_name] = sr
        return VMATResult(test_type=self._result_header, tolerance_percent=self._tolerance * 100, max_deviation_percent=self.max_r_deviation,
                          abs_mean_deviation=self.avg_abs_r_deviation, passed=self.passed, segment_data=segment_data,
                          named_segment_data=named)


@capture_warnings
class DRGS(VMATLinearBase):
    """vmat.py:843-869"""

    _result_header = "Dose Rate & Gantry Speed"
    _result_short_header = "DR/GS"

    @classmethod
    def _default_roi_config(cls) -> dict:
        return {"ROI 1": {"offset_mm": -60}, "ROI 2": {"offset_mm": -40}, "ROI 3": {"offset_mm": -20}, "ROI 4": {"offset_mm": 0},
                "ROI 5": {"offset_mm": 20}, "ROI 6": {"offset_mm": 40}, "ROI 7": {"offset_mm": 60}}


@capture_warnings
class DRMLC(VMATLinearBase):
    """vmat.py:872-895"""

    _result_header = "Dose Rate & MLC Speed"
    _result_short_header = "DR/MLCS"

    @classmethod
    def _default_roi_config(cls) -> dict:
        return {"ROI 1": {"offset_mm": -45}, "ROI 2": {"offset_mm": -15}, "ROI 3": {"offset_mm": 15}, "ROI 4": {"offset_mm": 45}}


@capture_warnings
class DRCS(VMATBase):
    """vmat.py:898-1313: dose rate vs collimator speed."""

    text_rotation = 0
    _result_header = "Dose Rate & Collimator Speed"
    _result_short_header = "DR/CS"
    _default_radial_distance = 50  # mm

    @property
    def default_segment_size_mm(self) -> tuple[float, float]:
        return 40, 10

    @property
    def default_roi_config(self) -> dict:
        d = self._default_radial_distance
        return {"ROI 1": {"radial_distance": d, "angle": -120}, "ROI 2": {"radial_distance": d, "angle": -60},
                "ROI 3": {"radial_distance": d, "angle": 0}, "ROI 4": {"radial_distance": d, "angle": 60},
                "ROI 5": {"radial_distance": d, "angle": 120}}

    @property
    def default_collimator_config(self) -> dict[str, float]:
        return {"A": 150, "B": 90, "C": 30, "D": 330, "E": 270, "F": 210}  # IEC

    @property
    def default_collimator_radial_distances(self) -> tuple[float, float]:
        return 30, 70  # mm

    @property
    def rotation_offset_deg(self) -> float:
        return float(np.mean([cd.angle_deviation for cd in self.collimator_deviations]))

    def _identify_images(self, image1, image2):
        """vmat.py:979-999: the image whose max-normalised 10 x 10 median has the larger sum is the open field (device median)."""
        sums = []
        ctx = nat.Context.default()
        for img in (image1, image2):
            tmp = image.ArrayImage(np.ascontiguousarray(frame_u16(img, "VMAT")))
            tmp.filter(size=10, kind="median")
            with nat.Batch.upload(ctx, tmp.array) as b:
                st = nat.frame_stats(ctx, b)       # exact integer sum and max of the filtered frame
            sums.append(float(st["sum"][0]) / float(st["max"][0]))       # normalize(...).sum()
        if sums[0] > sums[1]:
            self.open_image, self.dmlc_image = image1, image2
        else:
            self.open_image, self.dmlc_image = image2, image1

    def analyze(self, tolerance: float | int = 1.5, segment_size_mm: tuple | None = None, roi_config: dict | None = None,
                collimator_radial_distances: tuple[float, float] | None = None, collimator_config: dict | None = None,
                invert_image_order: bool = False):
        """vmat.py:937-977"""
        if segment_size_mm is None:
            segment_size_mm = self.default_segment_size_mm
        if roi_config is None:
            roi_config = self.default_roi_config
        if invert_image_order:
            self.open_image, self.dmlc_image = self.dmlc_image, self.open_image
        self._tolerance = tolerance / 100
        self.roi_config = roi_config
        self._ratio = None
        self.segments = []
        self._calculate_segments(segment_size_mm)
        self._update_r_corrs()
        cc = collimator_config or self.default_collimator_config
        crd = collimator_radial_distances or self.default_collimator_radial_distances
        self._calculate_collimator_deviations(cc, crd)

    def _calculate_segments(self, segment_size_mm):
        """vmat.py:1050-1082: EuclideanTransform(translation=(r, 0)) + rotation + translation(image centre), written out"""
        dpmm = self.open_image.dpmm
        cx, cy = self.open_image.center.x, self.open_image.center.y
        geo = []
        for roi_data in self.roi_config.values():
            r_px = roi_data["radial_distance"] * dpmm
            angle_rad = np.deg2rad(-roi_data["angle"] - 90)
            cs, sn = math.cos(angle_rad), math.sin(angle_rad)
            # composed matrix = T(centre) @ R(angle) @ T(r, 0): translation column and the rotation skimage reads back from it
            tx, ty = cs * r_px + cx, sn * r_px + cy
            rotation = math.atan2(sn, cs)
            geo.append((Point(tx, ty), segment_size_mm[0] * dpmm, segment_size_mm[1] * dpmm, float(np.rad2deg(rotation))))
        # the statistics of all segments in one device call: the ratio image is uploaded once, one CTA per segment
        rois = [RectangleROI(self.ratio_image, w, h, c, rot) for c, w, h, rot in geo]
        st = nat.roi_stats(nat.Context.default(), self.ratio_image, np.stack([r._polygon_xy() for r in rois]))
        for k, (c, w, h, rot) in enumerate(geo):
            self.segments.append(Segment(c, width=w, height=h, tolerance=self._tolerance, rotation=rot, r_corr=float(st["mean"][0, k]) * 100,
                                         stdev=float(st["std"][0, k])))

    def _calculate_collimator_deviations(self, collimator_config: dict[str, float], collimator_radial_distances):
        """vmat.py:1084-1149"""
        num_config_angles = len(collimator_config)
        if num_config_angles < 1:
            self.collimator_deviations = []
            return
        nominal_angles = np.fromiter(collimator_config.values(), dtype=float)
        sorted_angles = np.sort(nominal_angles)
        gaps = np.diff(sorted_angles)
        wrap_gap = (sorted_angles[0] + 360) - sorted_angles[-1]
        min_diff_angle = min(np.min(gaps), wrap_gap) if len(gaps) else wrap_gap
        crd_px = np.array(collimator_radial_distances) * self.dmlc_image.dpmm
        peaks = []
        for crd in crd_px:
            circle_profile = CircleProfile(center=self.dmlc_image.center, radius=crd, image_array=self.ratio_image, start_angle=math.pi / 2)
            min_distance = 2 * np.pi * crd / 360 * 0.9 * min_diff_angle
            circle_profile.find_peaks(min_distance=min_distance, threshold=0.8)
            peaks.append(circle_profile.peaks)
        if not peaks:
            raise ValueError("Could not detect collimator lines.")
        num_detected = len(peaks[0])
        if any(len(p) != num_detected for p in peaks):
            raise ValueError("Could not consistently detect collimator lines across radii. "
                             f"Detected {[len(p) for p in peaks]} peaks across radii.")
        if num_config_angles > num_detected:
            raise ValueError(f"Configured {num_config_angles} collimator spokes but only detected {num_detected}. Check image quality / "
                             "analysis settings or reduce collimator_config.")
        candidate_points = [[peaks[k][i] for k in range(len(peaks))] for i in range(num_detected)]
        measured_angles = np.array([CollimatorDeviation.calculate_angle_measured(pts[0], pts[1]) for pts in candidate_points], dtype=float)
        self.collimator_deviations = []
        for name, nominal in collimator_config.items():
            deltas = np.abs(wrap180(measured_angles - float(nominal)))
            pts = candidate_points[int(np.argmin(deltas))]
            self.collimator_deviations.append(CollimatorDeviation(name, float(nominal), (pts[0], pts[1])))

    def _generate_results_data(self) -> DRCSResult:
        """vmat.py:1001-1038"""
        segment_data, named = [], {}
        for segment, (roi_name, roi_data) in zip(self.segments, self.roi_config.items()):
            sr = SegmentResult(passed=segment.passed, r_corr=segment.r_corr, r_dev=segment.r_dev, center_x_y=(segment.center.x, segment.center.y),
                               x_position_mm=roi_data["radial_distance"], stdev=segment.stdev, angular_position_deg=roi_data["angle"])
            segment_data.append(sr)
            named[roi_name] = sr
        coll = {cd.name: CollimatorResult(angle_deviation=cd.angle_deviation, angle_nominal=cd.angle_nominal)
                for cd in self.collimator_deviations}
        return DRCSResult(test_type=self._result_header, tolerance_percent=self._tolerance * 100, max_deviation_percent=self.max_r_deviation,
                          abs_mean_deviation=self.avg_abs_r_deviation, passed=self.passed, segment_data=segment_data,
                          named_segment_data=named, rotation_offset_deg=self.rotation_offset_deg, collimator_data=coll)
