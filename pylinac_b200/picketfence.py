"""Picket-fence analysis -- drop-in for the hot path of ``pylinac.picketfence`` (reference file cited per item).

``PicketFence(image).analyze(**kw)`` keeps the reference's signature and result accessors; underneath, the whole
frame pipeline (crop view, noise check, inversion check, ground/normalise, orientation, picket search, per-leaf
windows, FWHM positions, line fits, errors) runs in CUDA (pylinac_b200/csrc/pf.cu) with batch = 1.
``analyze_batch(frames, ...)`` is the batched entry point the benchmark uses (one result per frame).

Out of scope (SURVEY.md section 2 row 4): plotting, PDF/QuAAC export, trajectory-log overlay (``log=``).
"""
from __future__ import annotations

import enum
import warnings
from collections.abc import Sequence
from pathlib import Path

import numpy as np

from . import _native as nat
from .core import image
from .core.geometry import Line, Point
from .core.warnings import capture_warnings
from .core.utilities import ResultBase, ResultsDataMixin, convert_to_enum

LEFT_MLC_PREFIX = "A"
RIGHT_MLC_PREFIX = "B"


class Orientation(enum.Enum):
    """picketfence.py:61-65"""

    UP_DOWN = "Up-Down"
    LEFT_RIGHT = "Left-Right"


class MLCArrangement:
    """picketfence.py:68-100"""

    def __init__(self, leaf_arrangement: list[tuple[int, float]], offset: float = 0):
        self.centers = []
        self.widths = []
        rolling_edge = 0
        for leaf_num, width in leaf_arrangement:
            self.centers += np.arange(start=rolling_edge + width / 2, stop=leaf_num * width + rolling_edge + width / 2,
                                      step=width).tolist()
            rolling_edge = self.centers[-1] + width / 2
            self.widths += [width] * leaf_num
        self.centers = [c - np.mean(self.centers) + offset for c in self.centers]

    @property
    def leaves(self) -> list[int]:
        return np.arange(1, len(self.centers) + 1, dtype=int)[::-1].tolist()


class MLC(enum.Enum):
    """picketfence.py:103-135"""

    MILLENNIUM = {"name": "Millennium", "arrangement": MLCArrangement([(10, 10), (40, 5), (10, 10)])}
    HD_MILLENNIUM = {"name": "HD Millennium", "arrangement": MLCArrangement([(14, 5), (32, 2.5), (14, 5)])}
    BMOD = {"name": "B Mod", "arrangement": MLCArrangement([(40, 4)])}
    AGILITY = {"name": "Agility", "arrangement": MLCArrangement([(80, 5)])}
    MLCI = {"name": "MLCi", "arrangement": MLCArrangement([(40, 10)])}
    HALCYON_DISTAL = {"name": "Halcyon distal", "arrangement": MLCArrangement([(28, 10)])}
    HALCYON_PROXIMAL = {"name": "Halcyon proximal", "arrangement": MLCArrangement([(29, 10)])}


def _get_mlc_arrangement(value) -> MLCArrangement:  # picketfence.py:331-342
    if isinstance(value, MLC):
        return value.value["arrangement"]
    if isinstance(value, MLCArrangement):
        return value
    if isinstance(value, str):
        return [m.value["arrangement"] for _, m in MLC.__members__.items() if m.value["name"] == value][0]
    raise TypeError("mlc must be an MLC, MLCArrangement or str")


class PFResult(ResultBase):
    """picketfence.py:138-201"""

    tolerance_mm: float
    action_tolerance_mm: float | None
    percent_leaves_passing: float
    number_of_pickets: int
    absolute_median_error_mm: float
    max_error_mm: float
    max_error_picket: int
    max_error_leaf: str | int
    mean_picket_spacing_mm: float
    offsets_from_cax_mm: list[float]
    passed: bool
    failed_leaves: list[str] | list[int]
    mlc_skew: float
    picket_widths: dict[str, dict[str, float]]
    mlc_positions_by_leaf: dict[str, list[float]]
    mlc_errors_by_leaf: dict[str, list[float]]
    cax: dict


STATUS_EXCEPTIONS = {
    1: (ValueError, "No pickets were found. This can mean either an incorrect orientation or incorrect inversion. "
                    "Try passing the correct orientation; if that fails, also set invert=True."),
    2: (ValueError, "No MLC measurements were found. This may be due to an incorrect inversion. Try setting invert=True. "
                    "Or, you may have passed an incorrect orientation."),
    3: (NotImplementedError, f"More than {nat.PF_MAX_PICKETS} pickets were detected; unsupported."),
    4: (IndexError, "An MLC window profile has no peak (the reference raises IndexError in FWXMProfile.field_edge_idx)."),
    5: (MemoryError, "Measurement table / window capacity exceeded."),
    6: (ValueError, "The image is flat (max == min); cannot normalize."),
    7: (TypeError, "expected non-empty vector for x (a picket has no MLC measurements)."),
    8: (ValueError, "cannot convert float NaN to integer (one picket was found, so the picket spacing is nan: pass picket_spacing)."),
}


def make_params(dpmm: float, shape, *, crop_mm=3, filter=None, mlc=MLC.MILLENNIUM, tolerance=0.5, action_tolerance=None,
                num_pickets=None, sag_adjustment=0, orientation=None, invert=False, leaf_analysis_width_ratio=0.4,
                picket_spacing=None, height_threshold=0.5, edge_threshold=1.5, peak_sort="peak_heights",
                required_prominence=0.2, fwxm=50, separate_leaves=False, nominal_gap_mm=3, central_axis=None) -> nat.PFParams:
    """Translate the reference's constructor + analyze() keyword arguments (picketfence.py:280-289, 636-654) into the
    C-ABI parameter block.  ``fwxm`` is accepted and ignored exactly like the reference does (it stores the value,
    picketfence.py:1563, but never forwards it to FWXMProfilePhysical, :1610-1615)."""
    if action_tolerance is not None and tolerance < action_tolerance:
        raise ValueError("Tolerance cannot be lower than the action tolerance")
    arr = _get_mlc_arrangement(mlc)
    n = len(arr.centers)
    if n > nat.PF_MAX_LEAVES:
        raise NotImplementedError(f"MLC arrangements with more than {nat.PF_MAX_LEAVES} leaves are not supported")
    p = nat.PFParams()
    p.dpmm = float(dpmm)
    p.crop_px = int(round(crop_mm * dpmm))
    p.filter_size = int(filter) if isinstance(filter, int) and not isinstance(filter, bool) else 0
    p.tolerance = float(tolerance)
    p.action_tolerance = -1.0 if action_tolerance is None else float(action_tolerance)
    p.num_pickets = int(num_pickets) if num_pickets else 0
    p.sag_px = int(round(sag_adjustment * dpmm)) if sag_adjustment != 0 else 0
    if orientation is None:
        p.orientation = -1
    else:
        p.orientation = 0 if convert_to_enum(orientation, Orientation) == Orientation.UP_DOWN else 1
    p.invert = 1 if invert else 0
    p.leaf_analysis_width_ratio = float(leaf_analysis_width_ratio)
    p.picket_spacing = -1.0 if picket_spacing is None else float(picket_spacing)
    p.height_threshold = float(height_threshold)
    p.edge_threshold = float(edge_threshold)
    p.peak_sort = 1 if peak_sort == "peak_heights" else 0
    p.required_prominence = -1.0 if required_prominence is None else float(required_prominence)
    p.separate_leaves = 1 if separate_leaves else 0
    p.nominal_gap_mm = float(nominal_gap_mm)
    if central_axis is not None:
        # PFDicomImage.center (picketfence.py:246-260) on the CROPPED image
        h = shape[0] - 2 * p.crop_px
        w = shape[1] - 2 * p.crop_px
        cx = (w / 2 - 0.5) + central_axis.x * dpmm
        cy = (h / 2 - 0.5) + central_axis.y * dpmm
        cy = 2 * (h // 2) - cy
        p.has_cax_override = 1
        p.cax_x_px = cx
        p.cax_y_px = cy
    p.n_leaves = n
    for i in range(n):
        p.leaf_center_mm[i] = float(arr.centers[i])
        p.leaf_width_mm[i] = float(arr.widths[i])
        p.leaf_num[i] = int(arr.leaves[i])
    return p


class PFFrameResult:
    """Lazy, per-frame view over the struct-of-arrays the GPU returned (no Python objects per MLC kiss until asked)."""

    def __init__(self, summary, meas, params: nat.PFParams, tolerance, action_tolerance, separate_leaves):
        self.s = summary
        self.m = meas[: int(summary["n_meas"])] if int(summary["status"]) == 0 else meas[:0]
        self.params = params
        self.tolerance = tolerance
        self.action_tolerance = action_tolerance
        self.separate_leaves = bool(separate_leaves)

    @property
    def status(self) -> int:
        return int(self.s["status"])

    def raise_for_status(self):
        if self.status:
            exc, msg = STATUS_EXCEPTIONS.get(self.status, (RuntimeError, f"picket fence status {self.status}"))
            raise exc(msg)

    @property
    def orientation(self) -> Orientation:
        return Orientation.UP_DOWN if int(self.s["orientation"]) == 0 else Orientation.LEFT_RIGHT

    @property
    def num_pickets(self) -> int:
        return int(self.s["n_pickets"])

    @property
    def picket_idx(self) -> np.ndarray:
        return self.s["picket_idx"][: self.num_pickets].astype(np.int64)

    def _npos(self):
        return 2 if self.separate_leaves else 1

    def _leaf_name(self, leaf, bank):
        if not self.separate_leaves:
            return int(leaf)
        return f"{LEFT_MLC_PREFIX if bank == 0 else RIGHT_MLC_PREFIX}{int(leaf)}"

    def failed_leaves(self):
        out = []
        for row in self.m:
            ok = [bool(row["passed"][k]) for k in range(self._npos())]
            if all(ok):
                continue
            names = [int(row["leaf_num"])] if not self.separate_leaves else [self._leaf_name(row["leaf_num"], k) for k in range(2) if not ok[k]]
            for nme in names:
                if nme not in out:
                    out.append(nme)
        return out

    @property
    def max_error_leaf(self):
        if not self.separate_leaves:
            return int(self.s["max_error_leaf"])
        return self._leaf_name(self.s["max_error_leaf"], int(self.s["max_error_bank"]))

    def results_data(self) -> PFResult:
        self.raise_for_status()
        s = self.s
        npk = self.num_pickets
        dpmm = self.params.dpmm
        cax_phys = float(s["cax_px"]) / dpmm
        positions, errors = {}, {}
        npos = self._npos()
        for row in self.m:  # leaf-major, picket-minor (picketfence.py:1329-1338)
            for k in range(npos):
                name = str(self._leaf_name(row["leaf_num"], k))
                positions.setdefault(name, []).append(cax_phys - float(row["position"][k]) / dpmm)
                errors.setdefault(name, []).append(float(row["error"][k]))
        h, w = int(s["height"]), int(s["width"])
        if self.params.has_cax_override:
            cax = {"x": self.params.cax_x_px, "y": self.params.cax_y_px, "z": 0}
        else:
            cax = {"x": w / 2 - 0.5, "y": h / 2 - 0.5, "z": 0}
        return PFResult(
            tolerance_mm=self.tolerance,
            action_tolerance_mm=self.action_tolerance,
            percent_leaves_passing=float(s["percent_passing"]),
            number_of_pickets=npk,
            absolute_median_error_mm=float(s["abs_median_error_mm"]),
            max_error_mm=float(s["max_error_mm"]),
            max_error_picket=int(s["max_error_picket"]),
            max_error_leaf=self.max_error_leaf,
            mean_picket_spacing_mm=float(s["mean_picket_spacing_mm"]),
            offsets_from_cax_mm=[float(v) for v in s["offsets_from_cax_mm"][:npk]],
            passed=bool(s["passed"]),
            failed_leaves=self.failed_leaves(),
            mlc_skew=float(s["mlc_skew"]),
            picket_widths={f"picket_{k}": {"max": float(s["picket_width_max"][k]), "mean": float(s["picket_width_mean"][k]),
                                           "median": float(s["picket_width_median"][k]), "min": float(s["picket_width_min"][k])}
                           for k in range(npk)},
            mlc_positions_by_leaf=dict(sorted(positions.items())),
            mlc_errors_by_leaf=dict(sorted(errors.items())),
            cax=cax,
        )


class PFBatchResult(Sequence):
    def __init__(self, summary, meas, params, tolerance, action_tolerance, separate_leaves):
        self.summary = summary
        self.meas = meas
        self.params = params
        self._args = (tolerance, action_tolerance, separate_leaves)

    def __len__(self):
        return len(self.summary)

    def __getitem__(self, i) -> PFFrameResult:
        return PFFrameResult(self.summary[i], self.meas[i], self.params, *self._args)


def analyze_batch(frames, dpmm: float, *, device: int | None = None, meas_cap: int | None = None, crop_mm=3, filter=None,
                  mlc=MLC.MILLENNIUM, **analyze_kwargs) -> PFBatchResult:
    """Batched ``PicketFence(frame, filter=, mlc=, crop_mm=).analyze(**analyze_kwargs)`` over frames[n, h, w] uint16.

    ``frames`` may be a host ndarray (chunked H2D copies overlapped with compute) or a device-resident
    ``_native.Batch``.  Returns one lazily materialised result per frame.
    """
    ctx = nat.Context.default(device)
    if isinstance(frames, nat.Batch):
        (n, h, w), dt = frames.shape_dtype
    else:
        frames = np.asarray(frames)
        if frames.ndim == 2:
            frames = frames[None]
        n, h, w = frames.shape
    params = make_params(dpmm, (h, w), crop_mm=crop_mm, filter=filter, mlc=mlc, **analyze_kwargs)
    # measurement-table rows per frame: 1024 covers the usual 60 leaf pairs x <= 17 pickets; a frame that needs more reports
    # status 5 and the batch is re-run once with the largest table the arrangement can fill (the reference has no such limit)
    cap = 1024 if meas_cap is None else int(meas_cap)
    summ, meas = nat.pf_analyze(ctx, frames, params, meas_cap=cap)
    cap_max = min(8192, params.n_leaves * nat.PF_MAX_PICKETS)
    if meas_cap is None and cap < cap_max and (summ["status"] == 5).any():
        summ, meas = nat.pf_analyze(ctx, frames, params, meas_cap=cap_max)
    return PFBatchResult(summ, meas, params, analyze_kwargs.get("tolerance", 0.5), analyze_kwargs.get("action_tolerance"),
                         analyze_kwargs.get("separate_leaves", False))


def analyze_files(paths, *, device: int | None = None, threads: int = 8, pinned: bool = True, **kwargs) -> PFBatchResult:
    """Batched ``PicketFence(path).analyze()`` over DICOM files: header-only parse, then every file's pixel bytes are read straight
    into one page-locked [n, rows, cols] array (``dicom.read_frames``: no intermediate copy between the page cache and the H2D
    DMA), then ``analyze_batch``.  As in ``image.frame_u16`` the STORED integers are analysed (order-flipped where RescaleSlope /
    PixelIntensityRelationshipSign make the displayed values a decreasing map of them); all files must share shape, stored dtype
    and dpmm.  The reference loads and analyses one file at a time (core/io.py:73-84, core/image.py:1431-1444)."""
    from . import dicom
    from .core import image

    paths = [str(p) for p in paths]
    headers0 = dicom.read_header(paths[0])
    shape = (len(paths), int(headers0["Rows"]), int(headers0["Columns"]))
    if headers0["PixelDtype"] != np.dtype("<u2"):
        raise ValueError(f"analyze_files takes 16-bit unsigned pixel data, got {headers0['PixelDtype']}; use PicketFence(path)")
    out = None
    if pinned:
        try:
            out = nat.pinned_empty(shape, np.uint16)
        except nat.NativeError:
            out = None
    frames, headers = dicom.read_frames(paths, out=out, threads=threads)
    dpmms = []
    for i, h in enumerate(headers):
        stub = image.DicomImage.__new__(image.DicomImage)
        stub.metadata, stub._sid, stub._dpi, stub._sad = h, None, None, 1000
        dpmms.append(stub.dpmm)
        slope, intercept, sign = h.get("RescaleSlope"), h.get("RescaleIntercept"), h.get("PixelIntensityRelationshipSign")
        decreasing = (sign == -1) != (slope is not None and intercept is not None and float(slope) < 0)
        if decreasing:      # exact modular order flip of the stored values (image.frame_u16)
            f = frames[i]
            frames[i] = (int(f.max()) + int(f.min()) - f.astype(np.int64)).astype(np.uint16)
    if any(d is None for d in dpmms):
        raise ValueError("DPI was not a tag in the image nor was it passed in. Please pass a DPI value")
    if max(dpmms) - min(dpmms) > 1e-12 * max(dpmms):
        raise ValueError("the files have different pixel sizes at isocentre; analyse them in groups of equal dpmm")
    return analyze_batch(frames, float(dpmms[0]), device=device, **kwargs)


class PFImageMixin:
    """PFDicomImage behaviour (picketfence.py:204-260) that is not pixel arithmetic: the CAX override."""

    _central_axis: Point | None = None


class _PicketView:
    """The parts of ``Picket`` (picketfence.py:1857-1923) user code reads: fit, skew(), dist2cax, mlc_meas."""

    def __init__(self, fit, dist2cax, meas):
        self.fit = np.poly1d(fit)
        self.dist2cax = dist2cax
        self.mlc_meas = meas

    def skew(self) -> float:
        return float(np.rad2deg(self.fit.coefficients[0]))


class _MLCValueView:
    """The parts of ``MLCValue`` (picketfence.py:1529-1743) that are data."""

    def __init__(self, row, npos, dpmm, leaf_center_px, leaf_width_px, ratio, orientation, separate):
        self.leaf_num = int(row["leaf_num"])
        self.picket_num = int(row["picket"])
        self.position = tuple(float(row["position"][k]) for k in range(npos))
        self.error = [float(row["error"][k]) for k in range(npos)]
        self.passed = [bool(row["passed"][k]) for k in range(npos)]
        self.field_width_mm = float(row["width_mm"])
        self._dpmm = dpmm
        self.leaf_center_px = leaf_center_px
        self.leaf_width_px = leaf_width_px
        self._analysis_ratio = ratio
        self._orientation = orientation
        self._separate_leaves = separate

    @property
    def position_mm(self):
        return [p / self._dpmm for p in self.position]

    @property
    def full_leaf_nums(self):
        if not self._separate_leaves:
            return [self.leaf_num]
        return [f"{LEFT_MLC_PREFIX}{self.leaf_num}", f"{RIGHT_MLC_PREFIX}{self.leaf_num}"]

    @property
    def max_abs_error(self) -> float:
        return float(np.max(np.abs(self.error)))

    @property
    def marker_lines(self) -> list[Line]:  # picketfence.py:1725-1743
        upper = self.leaf_center_px - self.leaf_width_px / 2 * self._analysis_ratio
        lower = self.leaf_center_px + self.leaf_width_px / 2 * self._analysis_ratio
        lines = []
        for p in self.position:
            if self._orientation == Orientation.UP_DOWN:
                lines.append(Line((p, upper), (p, lower)))
            else:
                lines.append(Line((upper, p), (lower, p)))
        return lines

    def __repr__(self):
        return f"Leaf: {self.leaf_num}, Picket: {self.picket_num}"


def _pf_loader(path, **kwargs):
    """What ``PFDicomImage(path, crop_mm=0, **kwargs)`` loads in from_multiple_images (picketfence.py:384-391): the un-cropped linac
    DICOM image (arrays / image objects go through the generic loader)."""
    if isinstance(path, (np.ndarray, image.BaseImage)):
        return image.load(path, **kwargs)
    return image.LinacDicomImage(path, **kwargs)


@capture_warnings
class PicketFence(ResultsDataMixin[PFResult]):
    """picketfence.py:263-329, 439-562, 636-845, 1292-1363 -- same constructor / analyze() signature."""

    def __init__(self, filename, filter: int | None = None, log: str | None = None, use_filename: bool = False,
                 mlc=MLC.MILLENNIUM, crop_mm: int = 3, image_kwargs: dict | None = None):
        if log is not None:
            raise NotImplementedError("trajectory-log overlay (log=) is outside the accelerated hot path")
        img_kwargs = dict(image_kwargs or {})
        self._central_axis = img_kwargs.pop("central_axis", None)
        if isinstance(filename, np.ndarray):
            self._raw = image.ArrayImage(filename, **img_kwargs)
        elif isinstance(filename, image.BaseImage):
            self._raw = filename
        else:
            self._raw = image.LinacDicomImage(filename, use_filenames=use_filename, **img_kwargs)
        if self._raw.dpmm is None:
            raise ValueError("The image has no dpmm; pass image_kwargs={'dpi': ..., 'sid': ...} for array input")
        self._filter = filter
        self._crop_mm = crop_mm
        self.mlc = _get_mlc_arrangement(mlc)
        self._mlc_arg = mlc
        self._is_analyzed = False
        self._result: PFFrameResult | None = None
        self._warnings: list = []

    @classmethod
    def from_bb_setup(cls, *args, bb_image, bb_diameter: float, **kwargs):
        """picketfence.py:402-437: find the CAX on a BB setup image first (windowed disk locator around the image centre, bright BB first,
        dark BB on failure) and override the picket-fence image's central axis with the BB's physical offset from the image centre."""
        from .metrics.image import SizedDiskLocator

        bb_image = image.load(bb_image)

        def _metrics(invert: bool):
            return SizedDiskLocator.from_center_physical(expected_position_mm=(0, 0), search_window_mm=(30 + bb_diameter, 30 + bb_diameter),
                                                         radius_mm=bb_diameter / 2, radius_tolerance_mm=bb_diameter * 0.1 + 1, invert=invert)

        try:
            caxs = bb_image.compute(metrics=_metrics(invert=True))
        except ValueError:
            caxs = bb_image.compute(metrics=_metrics(invert=False))
        cax_shift = caxs[0] - bb_image.center
        # physical units: the two images may differ in size / dpmm
        cax_physical_shift = Point(x=cax_shift.x / bb_image.dpmm, y=cax_shift.y / bb_image.dpmm)
        image_kwargs = dict(kwargs.pop("image_kwargs", None) or {})
        image_kwargs["central_axis"] = cax_physical_shift
        instance = cls(*args, **kwargs, image_kwargs=image_kwargs)
        instance._from_bb_setup = True
        instance._bb_image = bb_image
        return instance

    @classmethod
    def from_multiple_images(cls, path_list, stretch_each: bool = True, method: str = "mean", mlc=MLC.MILLENNIUM, **kwargs):
        """picketfence.py:357-400: superimpose several images (e.g. one picket each) and analyse the composite.  The reference
        combines un-cropped images, writes the composite to an in-memory DICOM (a full-range re-quantisation to the stored dtype,
        core/image.py:1480-1485) and constructs the PicketFence from that file; ``image._resaved`` reproduces the write / read
        pair, so the device pipeline receives the same stored integers the reference analyses.  ``crop_mm`` goes to the
        constructor only; the loader's ``use_filenames`` becomes the constructor's ``use_filename``."""
        crop_mm = kwargs.pop("crop_mm", 3)
        combined = image.load_multiples(path_list, stretch_each=stretch_each, method=method, loader=_pf_loader, **kwargs)
        use_filename = kwargs.pop("use_filenames", False)
        return cls(image._resaved(combined), mlc=mlc, use_filename=use_filename, crop_mm=crop_mm, **kwargs)

    # the frame the GPU analyses: uint16, un-cropped (the crop is a device-side view)
    def _frame_u16(self) -> np.ndarray:
        return image.frame_u16(self._raw, "GPU picket-fence")

    def analyze(self, tolerance: float = 0.5, action_tolerance: float | None = None, num_pickets: int | None = None,
                sag_adjustment: float | int = 0, orientation=None, invert: bool = False,
                leaf_analysis_width_ratio: float = 0.4, picket_spacing: float | None = None, height_threshold: float = 0.5,
                edge_threshold: float = 1.5, peak_sort: str = "peak_heights", required_prominence: float = 0.2,
                fwxm: int = 50, separate_leaves: bool = False, nominal_gap_mm: float = 3, central_axis: Point | None = None) -> None:
        """picketfence.py:636-845"""
        if action_tolerance is not None and tolerance < action_tolerance:
            raise ValueError("Tolerance cannot be lower than the action tolerance")
        self.tolerance = tolerance
        self.action_tolerance = action_tolerance
        self.leaf_analysis_width = leaf_analysis_width_ratio
        self.separate_leaves = separate_leaves
        if central_axis:
            self._central_axis = central_axis
        frame = self._frame_u16()
        dpmm = self._raw.dpmm
        batch = analyze_batch(frame, dpmm, crop_mm=self._crop_mm, filter=self._filter, mlc=self._mlc_arg, tolerance=tolerance,
                              action_tolerance=action_tolerance, num_pickets=num_pickets, sag_adjustment=sag_adjustment,
                              orientation=orientation, invert=invert, leaf_analysis_width_ratio=leaf_analysis_width_ratio,
                              picket_spacing=picket_spacing, height_threshold=height_threshold, edge_threshold=edge_threshold,
                              peak_sort=peak_sort, required_prominence=required_prominence, fwxm=fwxm,
                              separate_leaves=separate_leaves, nominal_gap_mm=nominal_gap_mm, central_axis=self._central_axis)
        res = batch[0]
        res.raise_for_status()
        self._result = res
        if int(res.s["n_leaves_removed"]) > 0:
            warnings.warn("Some leaves were removed from analysis because they were not detected for all pickets. If some valid "
                          "leaves are missing try adjusting height_threshold or edge_threshold")
        self._is_analyzed = True

    # ------------------------------------------------------------------ accessors (picketfence.py:439-562)
    def _need(self) -> PFFrameResult:
        if not self._is_analyzed:
            raise ValueError("It appears the PF image has not been analyzed yet. Use .analyze() first.")
        return self._result

    @property
    def orientation(self) -> Orientation:
        return self._need().orientation

    @property
    def passed(self) -> bool:
        return bool(self._need().s["passed"])

    @property
    def percent_passing(self) -> float:
        return float(self._need().s["percent_passing"])

    @property
    def max_error(self) -> float:
        return float(self._need().s["max_error_mm"])

    @property
    def max_error_picket(self) -> int:
        return int(self._need().s["max_error_picket"])

    @property
    def max_error_leaf(self):
        return self._need().max_error_leaf

    @property
    def abs_median_error(self) -> float:
        return float(self._need().s["abs_median_error_mm"])

    @property
    def num_pickets(self) -> int:
        return self._need().num_pickets

    @property
    def mean_picket_spacing(self) -> float:
        return float(self._need().s["mean_picket_spacing_mm"])

    def mlc_skew(self) -> float:
        return float(self._need().s["mlc_skew"])

    def failed_leaves(self):
        return self._need().failed_leaves()

    def picket_width_stat(self, picket: int, metric: str = "max") -> float:
        return float(self._need().s[f"picket_width_{metric}"][picket])

    @property
    def mlc_meas(self) -> list[_MLCValueView]:
        r = self._need()
        p = r.params
        n_axis = r.s["height"] if r.orientation == Orientation.UP_DOWN else r.s["width"]
        centers = {int(p.leaf_num[i]): (p.leaf_center_mm[i], p.leaf_width_mm[i]) for i in range(p.n_leaves)}
        out = []
        for row in r.m:
            c_mm, w_mm = centers[int(row["leaf_num"])]
            out.append(_MLCValueView(row, r._npos(), p.dpmm, c_mm * p.dpmm + n_axis / 2, w_mm * p.dpmm,
                                     p.leaf_analysis_width_ratio, r.orientation, r.separate_leaves))
        return out

    @property
    def pickets(self) -> list[_PicketView]:
        r = self._need()
        meas = self.mlc_meas
        return [_PicketView([float(r.s["fit_slope"][k]), float(r.s["fit_intercept"][k])], float(r.s["offsets_from_cax_mm"][k]),
                            [m for m in meas if m.picket_num == k]) for k in range(r.num_pickets)]

    def results(self, as_list: bool = False):
        """picketfence.py:1292-1311"""
        r = self._need()
        offsets = " ".join(f"{float(v):.1f}" for v in r.s["offsets_from_cax_mm"][: r.num_pickets])
        gantry = getattr(self._raw, "gantry_angle", 0.0)
        coll = getattr(self._raw, "collimator_angle", 0.0)
        results = [
            "Picket Fence Results:",
            f"Gantry Angle (\N{DEGREE SIGN}): {gantry:2.1f}",
            f"Collimator Angle (\N{DEGREE SIGN}): {coll:2.1f}",
            f"Tolerance (mm): {self.tolerance}",
            f"Leaves passing (%): {self.percent_passing:2.1f}",
            f"Absolute median error (mm): {self.abs_median_error:2.3f}mm",
            f"Mean picket spacing (mm): {self.mean_picket_spacing:2.1f}mmn",
            f"Picket offsets from CAX (mm): {offsets}",
            f"Max Error: {self.max_error:2.3f}mm on Picket: {self.max_error_picket}, Leaf: {self.max_error_leaf}",
            f"MLC Skew: {self.mlc_skew():2.3f} degrees",
        ]
        if self.failed_leaves():
            results.append(f"Failing leaves: {self.failed_leaves()}")
        return results if as_list else "\n".join(results)

    def _generate_results_data(self) -> PFResult:
        return self._need().results_data()
