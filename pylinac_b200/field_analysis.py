"""Field (flatness / symmetry) analysis -- drop-in for the hot path of ``pylinac.field_analysis`` (reference file cited per item).

``FieldAnalysis(image, filter=None, image_kwargs=None).analyze(**kw)`` keeps the reference's signature and result accessors;
underneath, the whole per-frame pipeline (histogram inversion check, beam-centre search on the row / column sums, strip
profiles, SingleProfile interpolation / normalisation / edge detection, penumbra, field sizes, slopes, protocol flatness and
symmetry) runs in CUDA (pylinac_b200/csrc/field.cu).  ``analyze_batch(frames, dpmm, ...)`` is the batched entry point.

Supported: interpolation NONE / LINEAR, edge detection FWHM / INFLECTION_DERIVATIVE, every normalisation, protocols NONE /
VARIAN / SIEMENS / ELEKTA; the central ROI statistics are device reductions (csrc/roi.cu).  Not on the GPU path: SPLINE
interpolation, INFLECTION_HILL, plotting / PDF export.  The ``top_*`` results are the exact vertex of the fitted parabola (the
reference's L-BFGS-B run is noise-limited, see DESIGN.md).
"""
from __future__ import annotations

import enum
import warnings
from collections.abc import Sequence

import numpy as np

from . import _native as nat
from .core import image
from .core.profile import Centering, Edge, Interpolation, Normalization, SingleProfile
from .core.utilities import ResultBase, ResultsDataMixin, convert_to_enum


class Protocol(enum.Enum):
    """field_analysis.py:233-289 (the calculation tables live in csrc/field.cu)."""

    NONE = "NONE"
    VARIAN = "VARIAN"
    SIEMENS = "SIEMENS"
    ELEKTA = "ELEKTA"


_PROTOCOL_CODE = {Protocol.NONE: 0, Protocol.VARIAN: 1, Protocol.SIEMENS: 2, Protocol.ELEKTA: 3}
_CENTERING_CODE = {Centering.MANUAL: 0, Centering.BEAM_CENTER: 1, Centering.GEOMETRIC_CENTER: 2}
_NORM_CODE = {Normalization.NONE: 0, Normalization.GEOMETRIC_CENTER: 1, Normalization.BEAM_CENTER: 2, Normalization.MAX: 3}
_RESULT_KEYS = ["top_penumbra_mm", "bottom_penumbra_mm", "left_penumbra_mm", "right_penumbra_mm", "geometric_center_index_x_y",
                "beam_center_index_x_y", "field_size_vertical_mm", "field_size_horizontal_mm", "beam_center_to_top_mm",
                "beam_center_to_bottom_mm", "beam_center_to_left_mm", "beam_center_to_right_mm", "cax_to_top_mm", "cax_to_bottom_mm",
                "cax_to_left_mm", "cax_to_right_mm", "top_position_index_x_y", "top_horizontal_distance_from_cax_mm",
                "top_vertical_distance_from_cax_mm", "top_horizontal_distance_from_beam_center_mm",
                "top_vertical_distance_from_beam_center_mm", "left_slope_percent_mm", "right_slope_percent_mm",
                "top_slope_percent_mm", "bottom_slope_percent_mm"]


# ---- protocol calculations on a SingleProfile (field_analysis.py:37-231): scalar host work on the device-computed field values
def flatness_dose_difference(profile, in_field_ratio: float = 0.8, **kwargs) -> float:
    """field_analysis.py:37-61"""
    ser = kwargs.get("slope_exclusion_ratio", 0.2)
    dmax = profile.field_calculation(in_field_ratio=in_field_ratio, calculation="max", slope_exclusion_ratio=ser)
    dmin = profile.field_calculation(in_field_ratio=in_field_ratio, calculation="min", slope_exclusion_ratio=ser)
    return 100 * abs(dmax - dmin) / (dmax + dmin)


def flatness_dose_ratio(profile, in_field_ratio: float = 0.8, **kwargs) -> float:
    """field_analysis.py:64-82"""
    dmax = profile.field_calculation(in_field_ratio=in_field_ratio, calculation="max")
    dmin = profile.field_calculation(in_field_ratio=in_field_ratio, calculation="min")
    return 100 * (dmax / dmin)


def symmetry_point_difference(profile, in_field_ratio: float, **kwargs) -> float:
    """field_analysis.py:97-119: the point difference of largest magnitude (first one on ties), signed."""
    field = profile.field_data(in_field_ratio=in_field_ratio, slope_exclusion_ratio=kwargs.get("slope_exclusion_ratio", 0.2))
    fv = np.asarray(field["field values"], dtype=np.float64)
    sym = 100 * (fv - fv[::-1]) / field["beam center value (@rounded)"]
    return float(sym[int(np.argmax(np.abs(sym)))])


def symmetry_pdq_iec(profile, in_field_ratio: float, **kwargs) -> float:
    """field_analysis.py:183-207: max(|lt/rt|, |rt/lt|) with the sign of the larger ratio; first maximum on ties."""
    field = profile.field_data(in_field_ratio=in_field_ratio, slope_exclusion_ratio=kwargs.get("slope_exclusion_ratio", 0.2))
    fv = np.asarray(field["field values"], dtype=np.float64)
    s1, s2 = fv / fv[::-1], fv[::-1] / fv
    sign = np.where(np.abs(s1) > np.abs(s2), np.sign(s1), np.sign(s2))
    sym = np.maximum(np.abs(s1), np.abs(s2)) * sign
    return float(sym[int(np.argmax(np.abs(sym)))])


def symmetry_area(profile, in_field_ratio: float, **kwargs) -> float:
    """field_analysis.py:210-225"""
    import math

    fv = np.asarray(profile.field_data(in_field_ratio=in_field_ratio,
                                       slope_exclusion_ratio=kwargs.get("slope_exclusion_ratio", 0.2))["field values"], dtype=np.float64)
    n = len(fv)
    left, right = np.sum(fv[: math.floor(n / 2)]), np.sum(fv[math.ceil(n / 2):])
    return float(100 * (left - right) / (left + right))


# field_analysis.py:233-289: the calculation table of each protocol
_PROTOCOL_CALCS = {
    Protocol.NONE: {},
    Protocol.VARIAN: {"symmetry": symmetry_point_difference, "flatness": flatness_dose_difference},
    Protocol.SIEMENS: {"symmetry": symmetry_area, "flatness": flatness_dose_difference},
    Protocol.ELEKTA: {"symmetry": symmetry_pdq_iec, "flatness": flatness_dose_ratio},
}


class FieldResult(ResultBase):
    """field_analysis.py:291-439 (without the central ROI statistics)."""

    protocol: str
    protocol_results: dict
    centering_method: str | None
    normalization_method: str | None
    interpolation_method: str | None
    edge_detection_method: str
    top_penumbra_mm: float
    bottom_penumbra_mm: float
    left_penumbra_mm: float
    right_penumbra_mm: float
    geometric_center_index_x_y: tuple[float, float]
    beam_center_index_x_y: tuple[float, float]
    field_size_vertical_mm: float
    field_size_horizontal_mm: float
    beam_center_to_top_mm: float
    beam_center_to_bottom_mm: float
    beam_center_to_left_mm: float
    beam_center_to_right_mm: float
    cax_to_top_mm: float
    cax_to_bottom_mm: float
    cax_to_left_mm: float
    cax_to_right_mm: float
    top_position_index_x_y: tuple[float, float]
    top_horizontal_distance_from_cax_mm: float
    top_vertical_distance_from_cax_mm: float
    top_horizontal_distance_from_beam_center_mm: float
    top_vertical_distance_from_beam_center_mm: float
    left_slope_percent_mm: float
    right_slope_percent_mm: float
    top_slope_percent_mm: float
    bottom_slope_percent_mm: float
    central_roi_mean: float = 0
    central_roi_max: float = 0
    central_roi_std: float = 0
    central_roi_min: float = 0


class _CentralROI:
    """RectangleROI statistics of the reference's ``central_roi`` (field_analysis.py:755-766): the rectangle between the vertical
    and the horizontal extraction strips, evaluated on the image as ``analyze()`` leaves it (i.e. after the histogram / manual
    inversions: for a uint16 image inverted an odd number of times the statistics of max + min - v follow from those of v)."""

    def __init__(self, frame_u16: np.ndarray, row, inverted: bool):
        from .core.geometry import Point
        from .core.roi import RectangleROI

        left, right = int(row["strip_cols"][0]), int(row["strip_cols"][1])
        upper, lower = int(row["strip_rows"][0]), int(row["strip_rows"][1])
        self.width = max(abs(left - right), 2)
        self.height = max(abs(upper - lower), 2)
        self.center = Point(self.width / 2 + left, self.height / 2 + upper)
        roi = RectangleROI(frame_u16, width=self.width, height=self.height, center=self.center)
        mean, std, mn, mx = roi.mean, roi.std, roi.min, roi.max
        if inverted:
            s = float(int(frame_u16.max()) + int(frame_u16.min()))      # array_utils.invert: -a + max + min
            mean, mn, mx = s - mean, s - mx, s - mn
        self.mean, self.std, self.min, self.max = mean, std, mn, mx
        self.pixel_value = mean


def make_params(dpmm: float, *, protocol=Protocol.VARIAN, centering=Centering.BEAM_CENTER, vert_position: float = 0.5,
                horiz_position: float = 0.5, vert_width: float = 0, horiz_width: float = 0, in_field_ratio: float = 0.8,
                slope_exclusion_ratio: float = 0.2, invert: bool = False, is_FFF: bool = False, penumbra=(20, 80),
                interpolation=Interpolation.LINEAR, interpolation_resolution_mm: float = 0.1, ground: bool = True,
                normalization_method=Normalization.BEAM_CENTER, edge_detection_method=Edge.INFLECTION_DERIVATIVE,
                edge_smoothing_ratio: float = 0.003, hill_window_ratio: float = 0.15) -> nat.FieldParams:
    """analyze() arguments (field_analysis.py:565-586) -> the C-ABI struct."""
    protocol = Protocol[protocol] if isinstance(protocol, str) else protocol
    edge = convert_to_enum(edge_detection_method, Edge)
    interp = convert_to_enum(interpolation, Interpolation)
    norm = convert_to_enum(normalization_method, Normalization)
    cent = convert_to_enum(centering, Centering)
    if is_FFF and edge == Edge.FWHM:
        warnings.warn("Using FWHM for an FFF beam is not advised. Consider using INFLECTION_DERIVATIVE or INFLECTION_HILL")
    if edge == Edge.INFLECTION_HILL or interp == Interpolation.SPLINE:
        raise NotImplementedError("Edge.INFLECTION_HILL / Interpolation.SPLINE go through analyze_batch's per-profile path")
    if slope_exclusion_ratio >= in_field_ratio or slope_exclusion_ratio >= 1.0:
        raise ValueError("The exclusion region must be smaller than the field ratio")
    if penumbra[0] > penumbra[1]:
        raise ValueError("Upper penumbra value must be larger than the lower penumbra value")
    p = nat.FieldParams()
    p.dpmm = float(dpmm)
    p.protocol = _PROTOCOL_CODE[protocol]
    p.centering = _CENTERING_CODE[cent]
    p.vert_position, p.horiz_position = float(vert_position), float(horiz_position)
    p.vert_width, p.horiz_width = float(vert_width), float(horiz_width)
    p.in_field_ratio, p.slope_exclusion_ratio = float(in_field_ratio), float(slope_exclusion_ratio)
    p.invert = 1 if invert else 0
    p.penumbra_lower, p.penumbra_upper = float(penumbra[0]), float(penumbra[1])
    p.interpolation = 0 if interp == Interpolation.NONE else 1
    p.interpolation_resolution_mm = float(interpolation_resolution_mm)
    p.ground = 1 if ground else 0
    p.normalization = _NORM_CODE[norm]
    p.edge = 0 if edge == Edge.FWHM else 1
    p.edge_smoothing_ratio = float(edge_smoothing_ratio)
    return p


class FieldFrameResult:
    """One frame's results (a row of the struct-of-arrays the GPU returns)."""

    def __init__(self, row, protocol: Protocol, extra: dict | None = None):
        self.r = row
        self.protocol = protocol
        self.extra = extra or {}          # Edge.INFLECTION_HILL adds the four *_penumbra_percent_mm entries (field_analysis.py:775-787)

    @property
    def status(self) -> int:
        return int(self.r["status"])

    def raise_for_status(self):
        if self.status == 1:
            raise IndexError("no field edges were found in a profile (the image is likely inverted or empty)")
        if self.status == 2:
            raise ValueError("the image is flat (max == min)")

    def results_dict(self) -> dict:
        out = {}
        for k in _RESULT_KEYS:
            v = self.r[k]
            out[k] = tuple(float(x) for x in v) if np.ndim(v) else float(v)
        out.update(self.extra)
        return out

    def protocol_results(self) -> dict:
        if self.protocol == Protocol.NONE:
            return {}
        return {k: float(self.r[k]) for k in ("symmetry_horizontal", "symmetry_vertical", "flatness_horizontal", "flatness_vertical")}


class FieldBatchResult(Sequence):
    def __init__(self, rows: np.ndarray, protocol: Protocol, extras: list | None = None):
        self.rows = rows
        self.protocol = protocol
        self.extras = extras

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, i) -> FieldFrameResult:
        return FieldFrameResult(self.rows[i], self.protocol, self.extras[i] if self.extras else None)


def _analyze_per_profile(ctx, frames: "nat.Batch", dpmm: float, kw: dict) -> FieldBatchResult:
    """Edge.INFLECTION_HILL and / or Interpolation.SPLINE (field_analysis.py:503-562, 703-864).

    The frame work stays on the device: histogram inversion check, centre determination and strip bounds come from the batched
    pipeline (they do not depend on the edge method or the interpolation), the strip profiles are the exact integer column / row
    sums of the strips (``epid_frame_stats`` views) divided by the strip width.  Each profile then goes through the
    ``SingleProfile`` engine (cubic pre-sampling and Hill fits prepared on the host, core/profile.py) and the results are
    assembled as ``_analyze`` does.  Four engine launches and four small fits per frame: a per-image path, not a throughput path."""
    protocol = kw.get("protocol", Protocol.VARIAN)
    protocol = Protocol[protocol] if isinstance(protocol, str) else protocol
    edge = convert_to_enum(kw.get("edge_detection_method", Edge.INFLECTION_DERIVATIVE), Edge)
    interp = convert_to_enum(kw.get("interpolation", Interpolation.LINEAR), Interpolation)
    base_kw = dict(kw, edge_detection_method=Edge.FWHM, interpolation=Interpolation.NONE, protocol=Protocol.NONE, is_FFF=False)
    base = nat.field_analyze(ctx, frames, make_params(dpmm, **base_kw))
    (n, h, w), _ = frames.shape_dtype
    in_field_ratio = kw.get("in_field_ratio", 0.8)
    ser = kw.get("slope_exclusion_ratio", 0.2)
    penumbra = kw.get("penumbra", (20, 80))
    sp_kw = dict(dpmm=dpmm, interpolation=interp, interpolation_resolution_mm=kw.get("interpolation_resolution_mm", 0.1),
                 ground=kw.get("ground", True), edge_detection_method=edge, edge_smoothing_ratio=kw.get("edge_smoothing_ratio", 0.003),
                 normalization_method=kw.get("normalization_method", Normalization.BEAM_CENTER),
                 hill_window_ratio=kw.get("hill_window_ratio", 0.15))
    full = nat.frame_stats(ctx, frames)
    rows = np.zeros(n, nat.FIELD_RESULT_DTYPE)
    extras = []
    strip_stats: dict = {}
    for i in range(n):
        row = rows[i]
        for k in ("hist_inverted", "strip_rows", "strip_cols"):
            row[k] = base[i][k]
        extras.append({})
        if int(base[i]["status"]) == 2:
            row["status"] = 2
            continue
        bottom, top = (int(v) for v in base[i]["strip_rows"])
        left, right = (int(v) for v in base[i]["strip_cols"])
        hv, vv = (bottom, 0, top - bottom, w), (0, left, h, right - left)
        for view in (hv, vv):                      # frames of one batch nearly always share their strips: one launch per distinct view
            if view not in strip_stats:
                strip_stats[view] = nat.frame_stats(ctx, frames, view=view)
        horiz = strip_stats[hv]["colsum"][i] / (top - bottom)
        vert = strip_stats[vv]["rowsum"][i] / (right - left)
        if bool(int(base[i]["hist_inverted"])) != bool(kw.get("invert", False)):
            s_ = float(full["max"][i]) + float(full["min"][i])       # array_utils.invert: -a + max + min, exact on integers
            horiz, vert = s_ - horiz, s_ - vert
        try:
            hp, vp = SingleProfile(horiz, **sp_kw), SingleProfile(vert, **sp_kw)
            row["profile_len"] = (len(hp.values), len(vp.values))
            v_pen, h_pen = vp.penumbra(*penumbra), hp.penumbra(*penumbra)
            row["top_penumbra_mm"], row["bottom_penumbra_mm"] = v_pen["left penumbra width (exact) mm"], v_pen["right penumbra width (exact) mm"]
            row["left_penumbra_mm"], row["right_penumbra_mm"] = h_pen["left penumbra width (exact) mm"], h_pen["right penumbra width (exact) mm"]
            if edge == Edge.INFLECTION_HILL:
                extras[i] = {"top_penumbra_percent_mm": abs(v_pen["left gradient (exact) %/mm"]),
                             "bottom_penumbra_percent_mm": abs(v_pen["right gradient (exact) %/mm"]),
                             "left_penumbra_percent_mm": abs(h_pen["left gradient (exact) %/mm"]),
                             "right_penumbra_percent_mm": abs(h_pen["right gradient (exact) %/mm"])}
            row["geometric_center_index_x_y"] = (hp.geometric_center()["index (exact)"], vp.geometric_center()["index (exact)"])
            row["beam_center_index_x_y"] = (hp.beam_center()["index (exact)"], vp.beam_center()["index (exact)"])
            v1, h1 = vp.field_data(1.0, ser), hp.field_data(1.0, ser)
            row["field_size_vertical_mm"], row["field_size_horizontal_mm"] = v1["width (exact) mm"], h1["width (exact) mm"]
            row["beam_center_to_top_mm"] = v1["left distance->beam center (exact) mm"]
            row["beam_center_to_bottom_mm"] = v1["right distance->beam center (exact) mm"]
            row["beam_center_to_left_mm"] = h1["left distance->beam center (exact) mm"]
            row["beam_center_to_right_mm"] = h1["right distance->beam center (exact) mm"]
            row["cax_to_top_mm"], row["cax_to_bottom_mm"] = v1["left distance->CAX (exact) mm"], v1["right distance->CAX (exact) mm"]
            row["cax_to_left_mm"], row["cax_to_right_mm"] = h1["left distance->CAX (exact) mm"], h1["right distance->CAX (exact) mm"]
            hf, vf = hp.field_data(in_field_ratio, ser), vp.field_data(in_field_ratio, ser)
            row["top_position_index_x_y"] = (hf['"top" index (exact)'], vf['"top" index (exact)'])
            row["top_horizontal_distance_from_cax_mm"], row["top_vertical_distance_from_cax_mm"] = hf['"top"->CAX (exact) mm'], vf['"top"->CAX (exact) mm']
            row["top_horizontal_distance_from_beam_center_mm"] = hf['"top"->beam center (exact) mm']
            row["top_vertical_distance_from_beam_center_mm"] = vf['"top"->beam center (exact) mm']
            row["left_slope_percent_mm"], row["right_slope_percent_mm"] = hf["left slope (%/mm)"], hf["right slope (%/mm)"]
            row["top_slope_percent_mm"], row["bottom_slope_percent_mm"] = vf["left slope (%/mm)"], vf["right slope (%/mm)"]
            for name, calc in _PROTOCOL_CALCS[protocol].items():
                row[f"{name}_horizontal"] = calc(hp, in_field_ratio, slope_exclusion_ratio=ser)
                row[f"{name}_vertical"] = calc(vp, in_field_ratio, slope_exclusion_ratio=ser)
        except IndexError:
            row["status"] = 1
    return FieldBatchResult(rows, protocol, extras)


def analyze_batch(frames, dpmm: float, *, device: int | None = None, filter: int | None = None, **kwargs) -> FieldBatchResult:
    """FieldAnalysis(frame, filter=filter).analyze(**kwargs) for every frame of ``frames`` (uint16 [n,h,w] ndarray or Batch)."""
    ctx = nat.Context.default(device)
    per_profile = (convert_to_enum(kwargs.get("edge_detection_method", Edge.INFLECTION_DERIVATIVE), Edge) == Edge.INFLECTION_HILL
                   or convert_to_enum(kwargs.get("interpolation", Interpolation.LINEAR), Interpolation) == Interpolation.SPLINE)
    params = None if per_profile else make_params(dpmm, **kwargs)
    protocol = kwargs.get("protocol", Protocol.VARIAN)
    protocol = Protocol[protocol] if isinstance(protocol, str) else protocol
    with nat.batch_for(ctx, frames, np.uint16) as frames:
        if filter:
            with frames._unary(nat.lib().epid_median_filter, int(filter)) as filtered:   # image.filter(size=filter) (field_analysis.py:466)
                if per_profile:
                    return _analyze_per_profile(ctx, filtered, dpmm, kwargs)
                rows = nat.field_analyze(ctx, filtered, params)
        elif per_profile:
            return _analyze_per_profile(ctx, frames, dpmm, kwargs)
        else:
            rows = nat.field_analyze(ctx, frames, params)
    return FieldBatchResult(rows, protocol)


class FieldAnalysis(ResultsDataMixin[FieldResult]):
    """field_analysis.py:442-472, 565-864, 866-983 -- same constructor / analyze() signature."""

    def __init__(self, path, filter: int | None = None, image_kwargs: dict | None = None):
        img_kwargs = image_kwargs or {}
        self._path = path
        if isinstance(path, np.ndarray):
            self.image = image.ArrayImage(path, **img_kwargs)
        elif isinstance(path, image.BaseImage):
            self.image = path
        else:
            self.image = image.load(path, **img_kwargs)
        self._filter = filter
        self._is_analyzed = False

    def _frame_u16(self) -> np.ndarray:
        return image.frame_u16(self.image, "GPU field-analysis")

    def analyze(self, protocol=Protocol.VARIAN, centering=Centering.BEAM_CENTER, vert_position: float = 0.5, horiz_position: float = 0.5,
                vert_width: float = 0, horiz_width: float = 0, in_field_ratio: float = 0.8, slope_exclusion_ratio: float = 0.2,
                invert: bool = False, is_FFF: bool = False, penumbra=(20, 80), interpolation=Interpolation.LINEAR,
                interpolation_resolution_mm: float = 0.1, ground: bool = True, normalization_method=Normalization.BEAM_CENTER,
                edge_detection_method=Edge.INFLECTION_DERIVATIVE, edge_smoothing_ratio: float = 0.003,
                hill_window_ratio: float = 0.15, **kwargs) -> None:
        """field_analysis.py:565-642"""
        if self.image.dpmm is None:
            raise ValueError("The image has no dpmm; pass image_kwargs={'dpi': ..., 'sid': ...} for array input")
        self._protocol = Protocol[protocol] if isinstance(protocol, str) else protocol
        self._centering = convert_to_enum(centering, Centering)
        self._norm = convert_to_enum(normalization_method, Normalization)
        self._interp = convert_to_enum(interpolation, Interpolation)
        self._edge = convert_to_enum(edge_detection_method, Edge)
        self._penumbra = penumbra
        res = analyze_batch(self._frame_u16(), self.image.dpmm, filter=self._filter, protocol=self._protocol, centering=centering,
                            vert_position=vert_position, horiz_position=horiz_position, vert_width=vert_width,
                            horiz_width=horiz_width, in_field_ratio=in_field_ratio, slope_exclusion_ratio=slope_exclusion_ratio,
                            invert=invert, is_FFF=is_FFF, penumbra=penumbra, interpolation=interpolation,
                            interpolation_resolution_mm=interpolation_resolution_mm, ground=ground,
                            normalization_method=normalization_method, edge_detection_method=edge_detection_method,
                            edge_smoothing_ratio=edge_smoothing_ratio, hill_window_ratio=hill_window_ratio)[0]
        res.raise_for_status()
        self._result = res
        self._results = res.results_dict()
        self._extra_results = res.protocol_results()
        # the reference mutates its image: check_inversion_by_histogram() in the constructor, invert() in analyze()
        inverted = bool(int(res.r["hist_inverted"])) != bool(invert)
        self.central_roi = _CentralROI(self._frame_u16(), res.r, inverted)
        self._results.update(central_roi_mean=self.central_roi.mean, central_roi_max=self.central_roi.max,
                             central_roi_std=self.central_roi.std, central_roi_min=self.central_roi.min)
        self._is_analyzed = True

    def results(self, as_str: bool = True):
        """field_analysis.py:866-955 (the numeric lines)."""
        if not self._is_analyzed:
            raise ValueError("Image is not analyzed yet. Use analyze() first.")
        r = self._results
        out = ["Field Analysis Results", "----------------------", f"File: {self._path if not isinstance(self._path, np.ndarray) else 'array'}",
               f"Protocol: {self._protocol.name}", f"Centering method: {self._centering.value}",
               f"Normalization method: {self._norm.value}", f"Interpolation: {self._interp.value}",
               f"Edge detection method: {self._edge.value}", "",
               f"Penumbra width ({self._penumbra[0]}/{self._penumbra[1]}):", f"Left: {r['left_penumbra_mm']:3.1f}mm",
               f"Right: {r['right_penumbra_mm']:3.1f}mm", f"Top: {r['top_penumbra_mm']:3.1f}mm", f"Bottom: {r['bottom_penumbra_mm']:3.1f}mm", "",
               "Field Size:", f"Horizontal: {r['field_size_horizontal_mm']:3.1f}mm", f"Vertical: {r['field_size_vertical_mm']:3.1f}mm", "",
               "CAX to edge distances:", f"CAX -> Top edge: {r['cax_to_top_mm']:3.1f}mm", f"CAX -> Bottom edge: {r['cax_to_bottom_mm']:3.1f}mm",
               f"CAX -> Left edge: {r['cax_to_left_mm']:3.1f}mm", f"CAX -> Right edge: {r['cax_to_right_mm']:3.1f}mm", ""]
        out += ["Central ROI stats:", f"Mean: {self.central_roi.mean}", f"Max: {self.central_roi.max}", f"Min: {self.central_roi.min}",
                f"Standard deviation: {self.central_roi.std}", ""]
        for name in ("symmetry", "flatness"):
            if f"{name}_horizontal" in self._extra_results:
                out += [f"Vertical {name}: {self._extra_results[name + '_vertical']:3.3f}",
                        f"Horizontal {name}: {self._extra_results[name + '_horizontal']:3.3f}", ""]
        return "\n".join(out) if as_str else out

    def _generate_results_data(self) -> FieldResult:
        if not self._is_analyzed:
            raise ValueError("Image is not analyzed yet. Use analyze() first.")
        return FieldResult(**self._results, protocol=self._protocol.name, centering_method=self._centering.value,
                           normalization_method=self._norm.value, interpolation_method=self._interp.value,
                           edge_detection_method=self._edge.value, protocol_results=self._extra_results)
