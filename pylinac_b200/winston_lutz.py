"""Winston-Lutz per-image (2-D) analysis -- drop-in for ``pylinac.winston_lutz.WinstonLutz2D`` (reference file cited per item).

``WinstonLutz2D(image, **kw).analyze(**kw)`` keeps the reference's signature and accessors; the per-frame pipeline (histogram
inversion check, edge clean-up, ground / normalize, field mask centre of mass, BB search over <= 50 thresholds with labelling,
region properties and the five detection predicates, field / BB matching, CAX->BB and CAX->EPID vectors) runs in CUDA
(pylinac_b200/csrc/wl.cu).  ``analyze_batch(frames, dpmm, ...)`` is the batched entry point (one result per frame).

Scope (SURVEY.md section 8, rows a28-a32): BB arrangement ISO, one field and one BB per image; ``WinstonLutz`` analyses a
whole set as one GPU batch and does the set-level solve (3-D BB / field positions, isocentre sizes, statistics) on the host
from the N result rows, as the reference does.  Out of scope here: multi-target arrangements, ``shift_vector`` virtual
shifts, plotting / PDF / QuAAC.

The reference delegates labelling and region properties to scikit-image, which is absent from the build container: the CUDA
kernels follow the published algorithms (see oracle/skimage_shim.py); that boundary is unpinned against skimage itself.
"""
from __future__ import annotations

import enum
import math
from collections.abc import Sequence

import numpy as np

from . import _native as nat
from .core import image
from .core.geometry import Point, Vector
from .core.warnings import capture_warnings
from .core.utilities import ResultBase, ResultsDataMixin

BB_ERROR_MESSAGE = (
    "Unable to locate the BB. Make sure the field edges do not obscure the BB, that there are no artifacts in the images, that "
    "the 'bb_size' parameter is close to reality, and that the BB is near the center (within 2cm). If this is a large-field "
    "image or kV image try setting 'low_density_bb' to True."
)  # winston_lutz.py:50-54

_STATUS_ERRORS = {
    nat.WL_NO_BB: BB_ERROR_MESSAGE,
    nat.WL_MISMATCH: "The number of detected fields and BBs do not match",                     # winston_lutz.py:743-746
    nat.WL_NO_FIELD: "No fields were detected",                                                # winston_lutz.py:747-748
    nat.WL_CAPACITY: "The BB search window, field or a candidate region exceeds the capacity of the GPU pipeline",
    nat.WL_FLAT_IMAGE: "The image is flat (max == min)",
}


class Axis(enum.Enum):
    """winston_lutz.py:422-429"""

    GANTRY = "Gantry"
    COLLIMATOR = "Collimator"
    COUCH = "Couch"
    GB_COMBO = "GB Combo"
    GBP_COMBO = "GBP Combo"
    EPID = "Epid"
    REFERENCE = "Reference"


class WinstonLutz2DResult(ResultBase):
    """winston_lutz.py:432-453 (points / vectors serialised as dicts)"""

    variable_axis: str
    bb_location: dict
    cax2epid_vector: dict
    cax2epid_distance: float
    cax2bb_vector: dict
    cax2bb_distance: float
    field_cax: dict


def wrap360(value: float) -> float:
    """core/utilities.py wrap360"""
    return value % 360


def is_close_degrees(angle1: float, angle2: float, delta: float = 1) -> bool:
    """core/utilities.py:170-188"""
    if delta < 0:
        raise ValueError("Delta must be positive")
    a1, a2 = wrap360(angle1), wrap360(angle2)
    simple = abs(a1 - a2)
    return min(simple, 360 - simple) <= delta


def variable_axis(gantry: float, coll: float, couch: float, *, snap_tolerance: float = 3, gantry_reference: float = 0,
                  collimator_reference: float = 0, couch_reference: float = 0) -> Axis:
    """winston_lutz.py:1073-1107"""
    G0 = is_close_degrees(gantry, gantry_reference, delta=snap_tolerance)
    B0 = is_close_degrees(coll, collimator_reference, delta=snap_tolerance)
    P0 = is_close_degrees(couch, couch_reference, delta=snap_tolerance)
    if G0 and B0 and not P0:
        return Axis.COUCH
    if G0 and P0 and not B0:
        return Axis.COLLIMATOR
    if P0 and B0 and not G0:
        return Axis.GANTRY
    if P0 and B0 and G0:
        return Axis.REFERENCE
    if P0:
        return Axis.GB_COMBO
    return Axis.GBP_COMBO


def make_params(dpmm: float, *, bb_size_mm: float = 5, low_density_bb: bool = False, open_field: bool = False,
                bb_proximity_mm: float = 20) -> nat.WlParams:
    """WinstonLutz2D.analyze() arguments (winston_lutz.py:1152-1164) -> the C-ABI struct."""
    if not dpmm > 0:
        raise ValueError("dpmm must be positive")
    if not bb_size_mm > 0:
        raise ValueError("bb_size_mm must be positive")
    p = nat.WlParams()
    p.dpmm = float(dpmm)
    p.bb_size_mm = float(bb_size_mm)
    p.low_density_bb = 1 if low_density_bb else 0
    p.open_field = 1 if open_field else 0
    p.bb_proximity_mm = float(bb_proximity_mm)
    return p


class WLFrameResult:
    """One frame's results (a row of the struct-of-arrays the GPU returns)."""

    def __init__(self, row, bb_shift_px=None, dpmm: float | None = None):
        self.r = row
        # virtual BB shift (WLBaseImage.analyze(shift_vector=...), winston_lutz.py:719-736): added to the detected BB, pixels
        self._shift = bb_shift_px
        self._dpmm = dpmm

    @property
    def status(self) -> int:
        return int(self.r["status"])

    def raise_for_status(self):
        if self.status != nat.WL_OK:
            raise ValueError(_STATUS_ERRORS.get(self.status, f"Winston-Lutz status {self.status}"))

    @property
    def shape(self) -> tuple[int, int]:
        return int(self.r["height"]), int(self.r["width"])

    @property
    def bb(self) -> Point:
        if self._shift is not None:
            return Point(float(self.r["bb_x"]) + self._shift[0], float(self.r["bb_y"]) + self._shift[1])
        return Point(float(self.r["bb_x"]), float(self.r["bb_y"]))

    @property
    def field_cax(self) -> Point:
        return Point(float(self.r["field_x"]), float(self.r["field_y"]))

    @property
    def epid(self) -> Point:
        return Point(float(self.r["epid_x"]), float(self.r["epid_y"]))

    @property
    def cax2bb_vector(self) -> Vector:
        if self._shift is not None:      # winston_lutz.py:1189-1192 on the shifted BB
            d = (self.bb - self.field_cax) / self._dpmm
            return Vector(d.x, d.y, d.z)
        return Vector(float(self.r["cax2bb_x"]), float(self.r["cax2bb_y"]), 0.0)

    @property
    def cax2bb_distance(self) -> float:
        if self._shift is not None:      # winston_lutz.py:1195-1198
            return self.field_cax.distance_to(self.bb) / self._dpmm
        return float(self.r["cax2bb_distance"])

    @property
    def cax2epid_vector(self) -> Vector:
        return Vector(float(self.r["cax2epid_x"]), float(self.r["cax2epid_y"]), 0.0)

    @property
    def cax2epid_distance(self) -> float:
        return float(self.r["cax2epid_distance"])


class WLBatchResult(Sequence):
    def __init__(self, rows: np.ndarray):
        self.rows = rows

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, i) -> WLFrameResult:
        return WLFrameResult(self.rows[i])


def analyze_batch(frames, dpmm: float, *, device: int | None = None, bb_size_mm: float = 5, low_density_bb: bool = False,
                  open_field: bool = False, bb_proximity_mm: float = 20) -> WLBatchResult:
    """WinstonLutz2D(...).analyze(**kw) for every frame of ``frames`` (uint16 [n,h,w] ndarray or a device-resident Batch)."""
    ctx = nat.Context.default(device)
    params = make_params(dpmm, bb_size_mm=bb_size_mm, low_density_bb=low_density_bb, open_field=open_field,
                         bb_proximity_mm=bb_proximity_mm)
    return WLBatchResult(nat.wl2d_analyze(ctx, frames, params))


def bb_projection_with_rotation(offset_left: float, offset_up: float, offset_in: float, gantry: float, couch: float = 0.0,
                                sad: float = 1000, machine_scale=None) -> tuple[float, float]:
    """winston_lutz.py:3401-3463: isoplane projection (left/right, sup/inf) of a point given by its phantom offsets.  The reference
    builds scipy's Rotation.from_euler("xyz", [-couch, 0, gantry]) (extrinsic: about x, then z) and applies it to (up, left, in);
    written out here."""
    if machine_scale is not None and machine_scale != MachineScale.IEC61217:
        gantry, _, couch = convert_scale(machine_scale, MachineScale.IEC61217, gantry, 0, couch)
    a, c = math.radians(-couch), math.radians(gantry)
    x, y, z = offset_up, offset_left, offset_in
    # Rx(a)
    y1, z1 = y * math.cos(a) - z * math.sin(a), y * math.sin(a) + z * math.cos(a)
    # Rz(c)
    x2, y2 = x * math.cos(c) - y1 * math.sin(c), x * math.sin(c) + y1 * math.cos(c)
    mag = sad / (sad - x2)
    return -(y2 * mag), z1 * mag


def _virtual_shift_px(shift_vector, dpmm: float, gantry: float, couch: float, sad: float, machine_scale) -> tuple[float, float]:
    """winston_lutz.py:719-736: the image-space displacement (pixels) a phantom shift produces for the BB of one image"""
    lat, sup_inf = bb_projection_with_rotation(offset_left=-shift_vector.x, offset_up=shift_vector.z, offset_in=shift_vector.y, sad=sad,
                                               gantry=gantry, couch=couch, machine_scale=machine_scale)
    return lat * dpmm, -(sup_inf * dpmm)


@capture_warnings
class WinstonLutz2D(ResultsDataMixin[WinstonLutz2DResult]):
    """winston_lutz.py:629-1231 -- same constructor keywords / analyze() signature for the single-image case."""

    def __init__(self, file, use_filenames: bool = False, **kwargs):
        if isinstance(file, np.ndarray):
            self.image = image.ArrayImage(file, **{k: v for k, v in kwargs.items() if k in ("dpi", "sid", "dtype")})
        elif isinstance(file, image.BaseImage):
            self.image = file
        elif image._is_dicom(file):
            # the reference's WinstonLutz2D IS a LinacDicomImage (winston_lutz.py:629, 1137): axis angles come from the tags,
            # gantry= / coll= / couch= override them
            self.image = image.LinacDicomImage(file, use_filenames=use_filenames, **kwargs)
        else:
            self.image = image.load(file, **{k: v for k, v in kwargs.items() if k in ("dpi", "sid", "dtype")})
        self.gantry_angle = float(kwargs["gantry"] if kwargs.get("gantry") is not None else getattr(self.image, "gantry_angle", 0.0) or 0.0)
        self.collimator_angle = float(kwargs["coll"] if kwargs.get("coll") is not None else getattr(self.image, "collimator_angle", 0.0) or 0.0)
        self.couch_angle = float(kwargs["couch"] if kwargs.get("couch") is not None else getattr(self.image, "couch_angle", 0.0) or 0.0)
        if self.image.dpmm is None:
            raise ValueError("DPI was not a tag in the image nor was it passed in. Please pass a DPI value")
        self._is_analyzed = False
        self._result: WLFrameResult | None = None
        self._snap_tolerance = 3.0
        self._gantry_reference = self._collimator_reference = self._couch_reference = 0.0

    def _frame_u16(self) -> np.ndarray:
        return image.frame_u16(self.image, "GPU Winston-Lutz")

    @property
    def dpmm(self) -> float:
        return self.image.dpmm

    def analyze(self, bb_size_mm: float = 5, low_density_bb: bool = False, open_field: bool = False, shift_vector=None,
                snap_tolerance: float = 3, gantry_reference: float = 0, collimator_reference: float = 0,
                couch_reference: float = 0, bb_proximity_mm: float = 20, machine_scale=None) -> None:
        """winston_lutz.py:1152-1183"""
        if snap_tolerance < 0:
            raise ValueError("Snap tolerance must be >= 0")
        self._snap_tolerance = snap_tolerance
        self._gantry_reference = gantry_reference
        self._collimator_reference = collimator_reference
        self._couch_reference = couch_reference
        # with a virtual shift the proximity test applies to the SHIFTED BB (find_bb_matches runs after the shift): the device finds
        # the BB without the test, the test is repeated here on the shifted point
        res = analyze_batch(self._frame_u16(), self.dpmm, bb_size_mm=bb_size_mm, low_density_bb=low_density_bb, open_field=open_field,
                            bb_proximity_mm=1e9 if shift_vector else bb_proximity_mm)[0]
        res.raise_for_status()
        if shift_vector:
            sad = float(getattr(self.image, "sad", 1000.0) or 1000.0)
            res = WLFrameResult(res.r, _virtual_shift_px(shift_vector, self.dpmm, self.gantry_angle, self.couch_angle, sad, machine_scale),
                                self.dpmm)
            if not res.epid.distance_to(res.bb) < bb_proximity_mm * self.dpmm:      # nominal position of the single BB = EPID centre
                raise ValueError(BB_ERROR_MESSAGE)
        self._result = res
        self._is_analyzed = True
        self.bb = res.bb
        self.field_cax = res.field_cax
        self.shape = res.shape

    def __repr__(self):
        return f"WLImage(gantry={self.gantry_angle:.1f}, coll={self.collimator_angle:.1f}, couch={self.couch_angle:.1f})"

    def _need(self) -> WLFrameResult:
        if self._result is None:
            raise ValueError("The image is not analyzed. Use .analyze() first.")
        return self._result

    @property
    def epid(self) -> Point:
        return self._need().epid

    @property
    def cax2bb_vector(self) -> Vector:
        return self._need().cax2bb_vector

    @property
    def cax2bb_distance(self) -> float:
        return self._need().cax2bb_distance

    @property
    def cax2epid_vector(self) -> Vector:
        return self._need().cax2epid_vector

    @property
    def cax2epid_distance(self) -> float:
        return self._need().cax2epid_distance

    @property
    def variable_axis(self) -> Axis:
        return variable_axis(self.gantry_angle, self.collimator_angle, self.couch_angle, snap_tolerance=self._snap_tolerance,
                             gantry_reference=self._gantry_reference, collimator_reference=self._collimator_reference,
                             couch_reference=self._couch_reference)

    def _generate_results_data(self) -> WinstonLutz2DResult:
        """winston_lutz.py:1215-1231"""
        r = self._need()

        def ser(p):
            return {"x": p.x, "y": p.y, "z": p.z}

        return WinstonLutz2DResult(variable_axis=self.variable_axis.value, cax2bb_vector=ser(r.cax2bb_vector),
                                   cax2epid_vector=ser(r.cax2epid_vector), cax2bb_distance=r.cax2bb_distance,
                                   cax2epid_distance=r.cax2epid_distance, bb_location=ser(r.bb), field_cax=ser(r.field_cax))


def cbct_frames(volume, ratio: float, *, device: int | None = None):
    """The four frames WinstonLutz.from_cbct analyses (winston_lutz.py:1465-1505), on the device, from a CT volume [N, H, W] of
    int16 / uint16 slices in sorted order and ratio = SliceThickness / PixelSpacing[0]: the maximum-intensity projections over rows
    and columns (epid_stack_mip), their slice axis resampled by ``zoom(p, (1, ratio), grid_mode=True, mode='nearest', order=1)``
    (epid_zoom on each projection row), then rot90 / fliplr, scipy's integer rounding and the uint16 bits array_to_dicom writes
    (epid_cbct_views).  Returns [(uint16 device Batch, set indices)] in the order of the reference's file names G=0, G=180, G=270,
    G=90 (top, bottom, left, right): one batch of 4 for square slices, else one per frame shape."""
    ctx = nat.Context.default(device)
    with nat.Batch.upload(ctx, volume) as vol:
        colmax, rowmax = nat.stack_mip(ctx, vol)
    src = np.asarray(volume).dtype
    zoom = nat.lib().epid_zoom        # arguments (ratio, 1, 3): order 1, mode 'nearest' | grid_mode
    with colmax, rowmax, colmax._unary(zoom, float(ratio), 1, 3) as zc, rowmax._unary(zoom, float(ratio), 1, 3) as zr:
        if zc.shape_dtype[0] == zr.shape_dtype[0]:
            return [(nat.cbct_views(ctx, zr, zc, src), [0, 1, 2, 3])]
        return [(nat.cbct_views(ctx, zr, None, src), [0, 1]), (nat.cbct_views(ctx, zc, None, src), [2, 3])]


# ---------------------------------------------------------------------------------------------------------------- set level
class MachineScale(enum.Enum):
    """core/scale.py:30-72 (axis conversions relative to IEC 61217)."""

    IEC61217 = "IEC61217"
    ELEKTA_IEC = "ELEKTA_IEC"
    VARIAN_IEC = "VARIAN_IEC"
    VARIAN_STANDARD = "VARIAN_STANDARD"


def _to_iec(scale: MachineScale, gantry: float, coll: float, rotation: float):
    if scale == MachineScale.IEC61217:
        return gantry, coll, rotation
    if scale in (MachineScale.ELEKTA_IEC, MachineScale.VARIAN_IEC):
        return gantry, coll, wrap360(-rotation)
    return wrap360(180 - gantry), wrap360(180 - coll), wrap360(180 - rotation)


def convert_scale(input_scale: MachineScale, output_scale: MachineScale, gantry: float, collimator: float, rotation: float):
    """core/scale.py:75-92: every conversion is its own inverse, so to-IEC followed by from-IEC."""
    g, c, r = _to_iec(input_scale, gantry, collimator, rotation)
    return _to_iec(output_scale, g, c, r)


def _cosd(deg: float) -> float:
    return math.cos(math.radians(deg))


def _sind(deg: float) -> float:
    return math.sin(math.radians(deg))


def solve_3d_shift_vector_from_2d_planes(xs, ys, thetas, phis, scale: MachineScale = MachineScale.IEC61217) -> Vector:
    """Low et al. equations 6-9 generalised (winston_lutz.py:3492-3577): least-squares (pseudo-inverse) solve of the 2 n x 3
    system built from the in-plane offsets and the gantry / couch angles in Varian Standard scale."""
    if not (len(xs) == len(ys) == len(thetas) == len(phis)):
        raise ValueError("The x, y, theta, and phi arrays must all be the same length.")
    n = len(xs)
    A = np.zeros((2 * n, 3))
    xi = np.zeros(2 * n)
    for i in range(n):
        th, _, ph = convert_scale(scale, MachineScale.VARIAN_STANDARD, thetas[i], 0, phis[i])
        A[2 * i, :] = [-_cosd(ph), -_sind(ph), 0]
        A[2 * i + 1, :] = [-_cosd(th) * _sind(ph), _cosd(th) * _cosd(ph), -_sind(th)]
        xi[2 * i] = ys[i]
        xi[2 * i + 1] = -xs[i]
    long, lat, vert = np.linalg.pinv(A).dot(xi).squeeze()
    return Vector(x=lat, y=-long, z=vert)


def solve_3d_position_from_2d_planes(xs, ys, thetas, phis, scale: MachineScale = MachineScale.IEC61217) -> Vector:
    """winston_lutz.py:3580-3590"""
    return -solve_3d_shift_vector_from_2d_planes(xs, ys, thetas, phis, scale)


def straight_ray(vector: Vector, gantry_angle: float):
    """winston_lutz.py:3463-3489: the 40 mm back-projection segment through ``vector`` for a gantry angle."""
    from .core.geometry import Line

    c, s = _cosd(gantry_angle), _sind(gantry_angle)
    p1 = Point(vector.x * c + 20 * s, vector.y, vector.x * -s + 20 * c)
    p2 = Point(vector.x * c - 20 * s, vector.y, vector.x * -s - 20 * c)
    return Line(p1, p2)


def max_distance_to_lines(p, lines) -> float:
    """winston_lutz.py:3395-3398"""
    point = Point(p[0], p[1], p[2])
    return max(line.distance_to(point) for line in lines)


class WinstonLutzResult(ResultBase):
    """winston_lutz.py:456-541"""

    max_2d_cax_to_bb_mm: float
    median_2d_cax_to_bb_mm: float
    mean_2d_cax_to_bb_mm: float
    max_2d_cax_to_epid_mm: float
    median_2d_cax_to_epid_mm: float
    mean_2d_cax_to_epid_mm: float
    gantry_3d_iso_diameter_mm: float
    coll_2d_iso_diameter_mm: float
    couch_2d_iso_diameter_mm: float
    gantry_coll_3d_iso_diameter_mm: float
    num_total_images: int
    num_gantry_images: int
    num_coll_images: int
    num_couch_images: int
    num_gantry_coll_images: int
    max_gantry_rms_deviation_mm: float
    max_epid_rms_deviation_mm: float
    max_coll_rms_deviation_mm: float
    max_couch_rms_deviation_mm: float
    bb_shift_vector: dict
    image_details: list[WinstonLutz2DResult]
    keyed_image_details: dict[str, WinstonLutz2DResult]


class _SetImage:
    """One image of an analysed set: the GPU result row + the axis values (the WinstonLutz2D accessors of the reference)."""

    def __init__(self, row: WLFrameResult, dpmm: float, gantry: float, coll: float, couch: float, refs):
        self.r = row
        self.dpmm = dpmm
        self.gantry_angle, self.collimator_angle, self.couch_angle = gantry, coll, couch
        self._refs = refs

    bb = property(lambda self: self.r.bb)
    field_cax = property(lambda self: self.r.field_cax)
    epid = property(lambda self: self.r.epid)
    cax2bb_vector = property(lambda self: self.r.cax2bb_vector)
    cax2bb_distance = property(lambda self: self.r.cax2bb_distance)
    cax2epid_vector = property(lambda self: self.r.cax2epid_vector)
    cax2epid_distance = property(lambda self: self.r.cax2epid_distance)

    @property
    def variable_axis(self) -> Axis:
        return variable_axis(self.gantry_angle, self.collimator_angle, self.couch_angle, **self._refs)

    # BBFieldMatch vectors in coordinate space (y flipped; winston_lutz.py:265-285)
    def _coord(self, a: Point, b: Point) -> Vector:
        return Vector((a.x - b.x) / self.dpmm, -((a.y - b.y) / self.dpmm), (a.z - b.z) / self.dpmm)

    @property
    def bb_field_vector_mm(self) -> Vector:
        return self._coord(self.bb, self.field_cax)

    @property
    def bb_epid_vector_mm(self) -> Vector:
        return self._coord(self.bb, self.epid)

    @property
    def field_epid_vector_mm(self) -> Vector:
        return self._coord(self.field_cax, self.epid)

    @property
    def bb_epid_distance_mm(self) -> float:
        """winston_lutz.py:292-295"""
        return self.epid.distance_to(self.bb) / self.dpmm

    @property
    def bb_to_field_projection(self):
        return straight_ray(self.bb_field_vector_mm, self.gantry_angle)

    def results_data(self) -> WinstonLutz2DResult:
        def ser(p):
            return {"x": p.x, "y": p.y, "z": p.z}

        return WinstonLutz2DResult(variable_axis=self.variable_axis.value, cax2bb_vector=ser(self.cax2bb_vector),
                                   cax2epid_vector=ser(self.cax2epid_vector), cax2bb_distance=self.cax2bb_distance,
                                   cax2epid_distance=self.cax2epid_distance, bb_location=ser(self.bb),
                                   field_cax=ser(self.field_cax))


@capture_warnings
class WinstonLutz(ResultsDataMixin[WinstonLutzResult]):
    """winston_lutz.py:1234-1611, 1614-1850, 2548-2609 -- a set of EPID images analysed as one batch on the GPU; the set-level
    quantities (3-D gantry isocentre, 2-D collimator / couch isocentres, BB shift vector, distance statistics) are scalar
    host work on N result rows, as in the reference.

    ``WinstonLutz(directory_or_paths)`` loads DICOM files like the reference; ``WinstonLutz.from_arrays(frames, axes, dpmm=)``
    takes frames already in memory (uint16 [n,h,w]) with one (gantry, collimator, couch) triple per frame;
    ``WinstonLutz.from_cbct(directory)`` builds four frames from a CBCT series on the device."""

    is_from_cbct: bool = False

    def __init__(self, directory, use_filenames: bool = False, axis_mapping: dict | None = None, axes_precision: int | None = None,
                 dpi: float | None = None, sid: float | None = None, missing_axis_value=0):
        import os

        if isinstance(directory, (list, tuple)):
            paths = [str(p) for p in directory]
        else:
            paths = sorted(os.path.join(directory, f) for f in os.listdir(directory) if not f.startswith("."))
        if len(paths) < 2:
            raise ValueError("<2 valid WL images were found in the folder/file or passed. Ensure you chose the correct folder/file")
        frames, axes, dpmm = [], [], None
        for pth in paths:
            img = image.LinacDicomImage(pth, use_filenames=use_filenames, axes_precision=axes_precision, missing_axis_value=missing_axis_value)
            key = os.path.basename(pth)
            if axis_mapping and not use_filenames and key in axis_mapping:   # winston_lutz.py:1293-1306
                axes.append(tuple(float(v) for v in axis_mapping[key]))
            else:
                axes.append((float(img.gantry_angle), float(img.collimator_angle), float(img.couch_angle)))
            frames.append(image.frame_u16(img, "GPU Winston-Lutz"))
            dpmm = img.dpmm if dpmm is None else dpmm
        self._setup(np.stack(frames), axes, dpmm)

    @classmethod
    def from_zip(cls, zfile, **kwargs):
        """winston_lutz.py:1397-1410: instantiate from a ZIP archive of the DICOM images (frames are read before the directory goes)."""
        with image.TemporaryZipDirectory(zfile) as tmp:
            return cls(image.retrieve_image_files(tmp), **kwargs)

    @classmethod
    def from_arrays(cls, frames: np.ndarray, axes, *, dpmm: float):
        self = cls.__new__(cls)
        self._setup(np.asarray(frames), [tuple(float(v) for v in a) for a in axes], float(dpmm))
        return self

    @classmethod
    def from_cbct_zip(cls, file, raw_pixels: bool = False, **kwargs):
        """winston_lutz.py:1426-1442: ``from_cbct`` on the contents of a ZIP archive."""
        with image.TemporaryZipDirectory(file) as tmp:
            return cls.from_cbct(tmp, raw_pixels=raw_pixels, **kwargs)

    @classmethod
    def from_cbct(cls, directory, raw_pixels: bool = False, **kwargs):
        """winston_lutz.py:1444-1509: a 4-angle Winston-Lutz set from a CBCT series.  The two maximum-intensity projections of the
        volume, their slice axis resampled to square pixels, are "viewed" from the left, top, right and bottom as gantry 270 / 0 / 90
        / 180 images; ``analyze()`` then forces ``low_density_bb`` and ``open_field``.  The volume goes to the GPU once
        (epid_stack_mip, epid_zoom, epid_cbct_views) and the four frames stay there for the analysis; no file is written.

        ``kwargs`` are WinstonLutz's (``use_filenames``, ``axis_mapping``, ``axes_precision``, ``missing_axis_value``; ``dpi`` / ``sid``
        are accepted as there) and resolve the axes of the images the reference writes: files ``G=270``, ``G=0``, ``G=90``,
        ``G=180`` with those gantry angles, collimator and couch 0.  Only integer frames are analysed: with ``raw_pixels=False`` a
        series whose rescale tags turn the slices into float Hounsfield units raises NotImplementedError; pass ``raw_pixels=True``
        (as the reference's docstring advises)."""
        stack = image.DicomImageStack(directory, min_number=10, raw_pixels=raw_pixels)
        return cls._from_stack(stack, **kwargs)

    @classmethod
    def _from_stack(cls, stack, use_filenames: bool = False, axis_mapping: dict | None = None, axes_precision: int | None = None,
                    dpi: float | None = None, sid: float | None = None, missing_axis_value=0):
        if any(im.array.dtype.kind == "f" or not np.may_share_memory(im.array, stack.volume) for im in stack.images):
            raise NotImplementedError("WinstonLutz.from_cbct analyses the stored integer slices only; this series' rescale turns them "
                                      "into other values. Pass raw_pixels=True.")
        md = stack.metadata
        pixel_mm = md.PixelSpacing[0]
        file_dpi = 25.4 / pixel_mm
        # array_to_dicom writes ImagePlanePixelSpacing = 25.4 / dpi, RTImageSID 1000 and RadiationMachineSAD 1000.0 (array_utils.py:281-283)
        dpmm = (1 / (25.4 / file_dpi)) * (1000 / 1000.0)
        names = sorted(f"G={g}" for g in (270, 0, 90, 180))       # the reference's file names, in this class's directory order
        axes = []
        for name in names:
            if axis_mapping and not use_filenames and name in axis_mapping:
                axes.append(tuple(float(v) for v in axis_mapping[name]))
                continue
            tags = {"gantry": float(f"{float(name[2:]):.2f}"), "coll": float(f"{0:.2f}"), "couch": float(f"{0:.2f}")}
            axes.append(tuple(image.linac_axis_value(key, None, name, tags[key], use_filenames=use_filenames,
                                                     missing_axis_value=missing_axis_value, axes_precision=axes_precision)
                              for key in ("gantry", "coll", "couch")))
        groups = cbct_frames(stack.volume, md.SliceThickness / pixel_mm)
        self = cls.__new__(cls)
        self._setup_groups(groups, axes, dpmm)
        self.is_from_cbct = True
        return self

    def _setup(self, frames: np.ndarray, axes, dpmm: float):
        if frames.ndim != 3 or len(axes) != frames.shape[0]:
            raise ValueError("frames must be [n,h,w] with one (gantry, collimator, couch) triple per frame")
        if frames.dtype != np.uint16:
            frames = image.frame_u16(frames, "GPU Winston-Lutz")
        self._setup_groups([(frames, list(range(len(axes))))], axes, dpmm)
        self._frames = frames

    def _setup_groups(self, groups, axes, dpmm: float):
        """groups: (uint16 frames [k,h,w] ndarray or device Batch, the set indices of those k images); one batch per frame shape"""
        self._groups, self._axes, self.dpmm = groups, axes, dpmm
        self.images: list[_SetImage] = []
        self._is_analyzed = False
        self.machine_scale = MachineScale.IEC61217
        self._minimized = {}
        self._virtual_shift = False

    def analyze(self, bb_size_mm: float = 5, machine_scale: MachineScale = MachineScale.IEC61217, low_density_bb: bool = False,
                open_field: bool = False, apply_virtual_shift: bool = False, snap_tolerance: float = 3, gantry_reference: float = 0,
                collimator_reference: float = 0, couch_reference: float = 0, bb_proximity_mm: float = 20) -> None:
        """winston_lutz.py:1519-1611"""
        self.machine_scale = machine_scale
        if self.is_from_cbct:      # winston_lutz.py:1564-1566
            low_density_bb = True
            open_field = True
        rows = [None] * len(self._axes)
        for frames, idx in self._groups:
            res = analyze_batch(frames, self.dpmm, bb_size_mm=bb_size_mm, low_density_bb=low_density_bb, open_field=open_field,
                                bb_proximity_mm=bb_proximity_mm)
            for j, k in enumerate(idx):
                rows[k] = res[j]
        refs = dict(snap_tolerance=snap_tolerance, gantry_reference=gantry_reference, collimator_reference=collimator_reference,
                    couch_reference=couch_reference)
        self.images = []
        for k, (g, c, p) in enumerate(self._axes):
            rows[k].raise_for_status()
            self.images.append(_SetImage(rows[k], self.dpmm, g, c, p, refs))
        self._minimized = {}
        if apply_virtual_shift:
            self._apply_virtual_shift(refs)
        self._bb_diameter = bb_size_mm
        self._is_analyzed = True

    def _apply_virtual_shift(self, refs: dict) -> None:
        """winston_lutz.py:1587-1601: the shift that would bring the BB to the radiation isocentre is applied to the detected BB of
        every image (the second pass of the reference re-detects the same BBs; its proximity default of 20 mm applies) and all
        set-level results are taken from the shifted BBs."""
        shift = self.bb_shift_vector
        self._virtual_shift = self.bb_shift_instructions()
        sad = float(getattr(self, "_sad", 1000.0))
        shifted = []
        for im in self.images:
            r = WLFrameResult(im.r.r, _virtual_shift_px(shift, self.dpmm, im.gantry_angle, im.couch_angle, sad, self.machine_scale), self.dpmm)
            if not r.epid.distance_to(r.bb) < 20 * self.dpmm:
                raise ValueError(BB_ERROR_MESSAGE)
            shifted.append(_SetImage(r, self.dpmm, im.gantry_angle, im.collimator_angle, im.couch_angle, refs))
        self.images = shifted
        self._minimized = {}

    # ---- BB3D (winston_lutz.py:313-362)
    def _solve(self, which: str) -> Point:
        vs = [getattr(m, which) for m in self.images]
        v = solve_3d_position_from_2d_planes([t.x for t in vs], [t.y for t in vs], [m.gantry_angle for m in self.images],
                                             [m.couch_angle for m in self.images], self.machine_scale)
        return Point(v.x, v.y, v.z)

    @property
    def measured_bb_position(self) -> Point:
        return self._solve("bb_epid_vector_mm")

    @property
    def measured_field_position(self) -> Point:
        return self._solve("field_epid_vector_mm")

    @property
    def bb_shift_vector(self) -> Vector:
        """winston_lutz.py:1703-1711"""
        d = self.measured_field_position - self.measured_bb_position
        return Vector(d.x, d.y, d.z)

    def bb_shift_instructions(self, couch_vrt: float | None = None, couch_lng: float | None = None,
                              couch_lat: float | None = None) -> str:
        """winston_lutz.py:1713-1745"""
        sv = self.bb_shift_vector
        x_dir = "LEFT" if sv.x < 0 else "RIGHT"
        y_dir = "IN" if sv.y > 0 else "OUT"
        z_dir = "UP" if sv.z > 0 else "DOWN"
        move = f"{x_dir} {abs(sv.x):2.2f}mm; {y_dir} {abs(sv.y):2.2f}mm; {z_dir} {abs(sv.z):2.2f}mm"
        if all(val is not None for val in [couch_vrt, couch_lat, couch_lng]):
            new_lat = round(couch_lat + sv.x / 10, 2)
            new_vrt = round(couch_vrt + sv.z / 10, 2)
            new_lng = round(couch_lng + sv.y / 10, 2)
            move += f"\nNew couch coordinates (cm): VRT: {new_vrt:3.2f}; LNG: {new_lng:3.2f}; LAT: {new_lat:3.2f}"
        return move

    # ---- isocentre sizes (winston_lutz.py:1614-1700)
    def _get_images(self, axis=(Axis.GANTRY,)):
        if isinstance(axis, Axis):
            axis = (axis,)
        imgs = [im for im in self.images if im.variable_axis in axis]
        return len(imgs), imgs

    def _minimize_axis(self, axes=(Axis.GANTRY,)):
        from scipy import optimize

        if isinstance(axes, Axis):
            axes = (axes,)
        if axes in self._minimized:
            return self._minimized[axes]
        things = [im.bb_to_field_projection for im in self.images if im.variable_axis in (axes + (Axis.REFERENCE,))]
        if len(things) <= 1:
            raise ValueError("Not enough images of the given type to identify the axis isocenter")
        result = optimize.minimize(max_distance_to_lines, np.array([0, 0, 0]), args=things, bounds=[(-20, 20)] * 3,
                                   options={"eps": 1e-7})
        self._minimized[axes] = result
        return result

    @property
    def gantry_iso_size(self) -> float:
        if self._get_images((Axis.GANTRY, Axis.REFERENCE))[0] > 1:
            return self._minimize_axis(Axis.GANTRY).fun * 2
        return 0

    @property
    def gantry_coll_iso_size(self) -> float:
        if self._get_images((Axis.GANTRY, Axis.COLLIMATOR, Axis.GB_COMBO, Axis.REFERENCE))[0] > 1:
            return self._minimize_axis((Axis.GANTRY, Axis.COLLIMATOR, Axis.GB_COMBO)).fun * 2
        return 0

    @staticmethod
    def _find_max_distance_between_points(images) -> float:
        pts = [Point(im.cax2bb_vector.x, im.cax2bb_vector.y) for im in images]
        return max(p1.distance_to(p2) for p1 in pts for p2 in pts)

    @property
    def collimator_iso_size(self) -> float:
        n, imgs = self._get_images((Axis.COLLIMATOR, Axis.REFERENCE))
        return self._find_max_distance_between_points(imgs) if n > 1 else 0

    @property
    def couch_iso_size(self) -> float:
        n, imgs = self._get_images((Axis.COUCH, Axis.REFERENCE))
        return self._find_max_distance_between_points(imgs) if n > 1 else 0

    def axis_rms_deviation(self, axis=Axis.GANTRY, value: str = "all"):
        """winston_lutz.py:1747-1774"""
        if isinstance(axis, (tuple, list)):
            axis = tuple(Axis(a) if not isinstance(a, Axis) else a for a in axis)
        elif not isinstance(axis, Axis):
            axis = Axis(axis)
        attr = "cax2bb_vector"
        if axis == Axis.EPID:
            attr = "cax2epid_vector"
            axis = (Axis.GANTRY, Axis.COLLIMATOR, Axis.REFERENCE)
        imgs = self._get_images(axis=axis)[1]
        if len(imgs) <= 1:
            return (0,)
        rms = [getattr(im, attr).as_scalar() for im in imgs]
        if value == "range":
            rms = max(rms) - min(rms)
        return rms

    def _metric(self, values, metric: str) -> float:
        import statistics

        if metric == "max":
            return max(values)
        if metric == "median":
            return statistics.median(values)
        if metric == "mean":
            return statistics.mean(values)
        raise ValueError("metric must be one of 'max', 'median', 'mean'")

    def cax2bb_distance(self, metric: str = "max") -> float:
        """winston_lutz.py:1776-1792"""
        return self._metric([im.cax2bb_distance for im in self.images], metric)

    def cax2epid_distance(self, metric: str = "max") -> float:
        """winston_lutz.py:1794-1810 -- as in the reference this aggregates ``epid_to_bb_distances()`` (EPID centre to BB,
        winston_lutz.py:838-843), not the per-image CAX-to-EPID distance."""
        return self._metric([im.bb_epid_distance_mm for im in self.images], metric)

    def results(self, as_list: bool = False):
        """winston_lutz.py:2501-2546: the text summary of an analysed set."""
        if not self._is_analyzed:
            raise ValueError("The set is not analyzed. Use .analyze() first.")
        num_gantry_imgs = self._get_images(axis=(Axis.GANTRY, Axis.REFERENCE))[0]
        num_gantry_coll_imgs = self._get_images(axis=(Axis.GANTRY, Axis.COLLIMATOR, Axis.GB_COMBO, Axis.REFERENCE))[0]
        num_coll_imgs = self._get_images(axis=(Axis.COLLIMATOR, Axis.REFERENCE))[0]
        num_couch_imgs = self._get_images(axis=(Axis.COUCH, Axis.REFERENCE))[0]
        num_imgs = len(self.images)
        result = [
            "Winston-Lutz Analysis",
            "=================================",
            f"Number of images: {num_imgs}",
            f"Maximum 2D CAX->BB distance: {self.cax2bb_distance('max'):.2f}mm",
            f"Median 2D CAX->BB distance: {self.cax2bb_distance('median'):.2f}mm",
            f"Mean 2D CAX->BB distance: {self.cax2bb_distance('mean'):.2f}mm",
        ]
        if getattr(self, "_virtual_shift", False):
            result.append(f"Virtual shift applied to BB to place at isocenter: {self._virtual_shift}")
        else:
            result.append(f"Shift to iso: facing gantry, move BB: {self.bb_shift_instructions()}")
        result += [
            f"Gantry 3D isocenter diameter: {self.gantry_iso_size:.2f}mm ({num_gantry_imgs}/{num_imgs} images considered)",
            f"Maximum Gantry RMS deviation (mm): {max(self.axis_rms_deviation((Axis.GANTRY, Axis.REFERENCE))):.2f}mm",
            f"Maximum EPID RMS deviation (mm): {max(self.axis_rms_deviation(Axis.EPID)):.2f}mm",
            f"Gantry+Collimator 3D isocenter diameter: {self.gantry_coll_iso_size:.2f}mm ({num_gantry_coll_imgs}/{num_imgs} images considered)",
            f"Collimator 2D isocenter diameter: {self.collimator_iso_size:.2f}mm ({num_coll_imgs}/{num_imgs} images considered)",
            f"Maximum Collimator RMS deviation (mm): {max(self.axis_rms_deviation((Axis.COLLIMATOR, Axis.REFERENCE))):.2f}",
            f"Couch 2D isocenter diameter: {self.couch_iso_size:.2f}mm ({num_couch_imgs}/{num_imgs} images considered)",
            f"Maximum Couch RMS deviation (mm): {max(self.axis_rms_deviation((Axis.COUCH, Axis.REFERENCE))):.2f}",
        ]
        return result if as_list else "\n".join(result)

    def _generate_results_data(self) -> WinstonLutzResult:
        """winston_lutz.py:2548-2609"""
        if not self._is_analyzed:
            raise ValueError("The set is not analyzed. Use .analyze() first.")
        details = [im.results_data() for im in self.images]
        keyed = {}
        for k, im in enumerate(self.images):
            key = f"G{im.gantry_angle}B{im.collimator_angle}P{im.couch_angle}"
            suffix, idx = "", 1
            while key + suffix in keyed:
                suffix = f"_{idx}"
                idx += 1
            keyed[key + suffix] = details[k]
        sv = self.bb_shift_vector
        return WinstonLutzResult(
            num_total_images=len(self.images),
            num_gantry_images=self._get_images((Axis.GANTRY, Axis.REFERENCE))[0],
            num_coll_images=self._get_images((Axis.COLLIMATOR, Axis.REFERENCE))[0],
            num_gantry_coll_images=self._get_images((Axis.GANTRY, Axis.COLLIMATOR, Axis.GB_COMBO, Axis.REFERENCE))[0],
            num_couch_images=self._get_images((Axis.COUCH, Axis.REFERENCE))[0],
            max_2d_cax_to_bb_mm=self.cax2bb_distance("max"), median_2d_cax_to_bb_mm=self.cax2bb_distance("median"),
            mean_2d_cax_to_bb_mm=self.cax2bb_distance("mean"), max_2d_cax_to_epid_mm=self.cax2epid_distance("max"),
            median_2d_cax_to_epid_mm=self.cax2epid_distance("median"), mean_2d_cax_to_epid_mm=self.cax2epid_distance("mean"),
            coll_2d_iso_diameter_mm=self.collimator_iso_size, couch_2d_iso_diameter_mm=self.couch_iso_size,
            gantry_3d_iso_diameter_mm=self.gantry_iso_size, gantry_coll_3d_iso_diameter_mm=self.gantry_coll_iso_size,
            max_gantry_rms_deviation_mm=max(self.axis_rms_deviation((Axis.GANTRY, Axis.REFERENCE))),
            max_coll_rms_deviation_mm=max(self.axis_rms_deviation((Axis.COLLIMATOR, Axis.REFERENCE))),
            max_couch_rms_deviation_mm=max(self.axis_rms_deviation((Axis.COUCH, Axis.REFERENCE))),
            max_epid_rms_deviation_mm=max(self.axis_rms_deviation(Axis.EPID)),
            bb_shift_vector={"x": sv.x, "y": sv.y, "z": sv.z}, image_details=details, keyed_image_details=keyed)
