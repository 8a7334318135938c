"""Field analysis via profiles and metric plug-ins -- drop-in for ``pylinac.field_profile_analysis.FieldProfileAnalysis``
(field_profile_analysis.py:90-220, 307-368) on top of the GPU primitives.

What runs on the GPU: the histogram inversion check, the row / column sums of the frame (field centre), the strip sums that
become the x / y profiles (exact integer sums of the uint16 pixels, one ``epid_frame_stats`` call per strip), the FWXM peak
search and the gaussian smoothing of the edge search.  The metric formulas (flatness, symmetry, penumbra, CAX distances:
``pylinac_b200/metrics/profile.py``) are scalar host arithmetic on the few hundred in-field samples of the two profiles.

Edge types: FWHM, INFLECTION_DERIVATIVE (the reference's default; its scipy minimisation of the cubic interpolant is replaced by the
closed-form stationary point of the same spline) and INFLECTION_HILL (4-parameter Hill fits of the two penumbrae, core/hill.py).
The central ROI statistics (``center_rect``) are one ``epid_roi_stats`` launch (core/roi.py).

``analyze_batch(frames, dpmm, ...)`` is the batched entry point: the frame-level device work (histogram inversion check, row /
column sums, strip sums, central ROI) is done for the whole batch in a handful of launches; the metric plug-ins are Python objects
by contract (``ProfileMetric.calculate``), so the per-frame profile objects are built on the host from the device-computed profiles.
"""
from __future__ import annotations

import copy
from collections.abc import Sequence

import numpy as np

from . import _native as nat
from .core import image
from .core.geometry import Point, Rectangle
from .core.profile import (Centering, Edge, FWXMProfilePhysical, HillProfilePhysical, InflectionDerivativeProfilePhysical,
                           Normalization)
from .core.roi import RectangleROI
from .core.warnings import capture_warnings
from .core.utilities import ResultBase, ResultsDataMixin, convert_to_enum
from .metrics.profile import (CAXToLeftEdgeMetric, CAXToRightEdgeMetric, FlatnessDifferenceMetric, PenumbraLeftMetric,
                              PenumbraRightMetric, ProfileMetric, SymmetryPointDifferenceMetric)


class FieldProfileResult(ResultBase):
    """field_profile_analysis.py:33-71"""

    x_metrics: dict
    y_metrics: dict
    center: dict
    normalization: str
    edge_type: str
    centering: str


def default_metrics() -> tuple[ProfileMetric, ...]:
    """field_profile_analysis.py:73-80 (fresh instances: a metric object keeps the profile it was injected into)."""
    return (FlatnessDifferenceMetric(), SymmetryPointDifferenceMetric(), PenumbraRightMetric(), PenumbraLeftMetric(),
            CAXToLeftEdgeMetric(), CAXToRightEdgeMetric())


PROFILES = {Edge.FWHM: FWXMProfilePhysical, Edge.INFLECTION_DERIVATIVE: InflectionDerivativeProfilePhysical,
            Edge.INFLECTION_HILL: HillProfilePhysical}


class NotAnalyzed(Exception):
    pass


@capture_warnings
class FieldProfileAnalysis(ResultsDataMixin[FieldProfileResult]):
    """field_profile_analysis.py:90-368 -- same constructor / analyze() keywords."""

    def __init__(self, path, **kwargs):
        if isinstance(path, np.ndarray):
            self.image = image.ArrayImage(path, **kwargs)
        elif isinstance(path, image.BaseImage):
            self.image = path
        else:
            self.image = image.load(path, **kwargs)
        self._is_analyzed = False
        self.image.check_inversion_by_histogram()

    # ---- device helpers: exact integer sums of frame strips
    def _frame_u16(self) -> np.ndarray:
        return image.frame_u16(self.image, "GPU field-profile")

    def analyze(self, centering=Centering.BEAM_CENTER, position: tuple[float, float] = (0.5, 0.5), x_width: float = 0.0,
                y_width: float = 0.0, normalization=Normalization.NONE, edge_type=Edge.INFLECTION_DERIVATIVE, invert: bool = False,
                ground: bool = True, metrics: Sequence[ProfileMetric] | None = None, **kwargs) -> None:
        """field_profile_analysis.py:123-194"""
        if invert:
            self.image.invert()
            self._flipped = not getattr(self, "_flipped", False)
        self._normalization = convert_to_enum(normalization, Normalization)
        self._edge_type = convert_to_enum(edge_type, Edge)
        self._centering = convert_to_enum(centering, Centering)
        metrics = default_metrics() if metrics is None else metrics
        ctx = nat.Context.default()
        frames = self._shared[0].batch if hasattr(self, "_shared") else self._frame_u16()
        with nat.batch_for(ctx, frames) as batch:
            x_values, y_values = self._get_profile_values(ctx, batch, position, x_width, y_width)
        cls = PROFILES[self._edge_type]
        self.x_profile = cls(values=x_values, dpmm=self.image.dpmm, normalization=normalization, ground=ground, **kwargs)
        self.x_profile.compute(metrics=metrics)
        self.y_profile = cls(values=y_values, dpmm=self.image.dpmm, normalization=normalization, ground=ground, **kwargs)
        self.y_profile.compute(metrics=copy.deepcopy(metrics))
        self._is_analyzed = True

    def _frame_sums(self, ctx, batch, view=None):
        """(column sums, row sums) of this object's frame over ``view`` = (row0, col0, rows, cols): exact integer sums from
        ``epid_frame_stats``.  Inside ``analyze_batch`` the launch covers the whole batch (shared per distinct view) and an inverted
        image (``-a + max + min``, exact on integers) is accounted for on the sums instead of re-uploading the flipped frame."""
        shared = getattr(self, "_shared", None)
        if shared is None:
            st = nat.frame_stats(ctx, batch, view=view)
            return st["colsum"][0], st["rowsum"][0]
        stats, i = shared
        st = stats.view(view) if view is not None else stats.full
        col, row = st["colsum"][i], st["rowsum"][i]
        if getattr(self, "_flipped", False):
            h, w = self.image.shape
            _, _, vh, vw = view if view is not None else (0, 0, h, w)
            s_ = float(stats.full["max"][i]) + float(stats.full["min"][i])
            col, row = s_ * vh - col, s_ * vw - row
        return col, row

    def _get_profile_values(self, ctx, batch, position, x_width, y_width):
        """field_profile_analysis.py:307-341: strips around (x, y); mean over the strip = exact integer sum / row count"""
        h, w = self.image.shape
        x, y = self._get_x_y_position(ctx, batch, position)
        if x_width > 1 or x_width < 0 or y_width > 1 or y_width < 0:
            raise ValueError("Width must be between 0 and 1")
        top = round(y - h * x_width / 2 - 1)
        bottom = round(max(y + h * x_width / 2, top + 2))
        left = round(x - w * y_width / 2 - 1)
        right = round(max(x + w * y_width / 2, left + 2))
        t, b = max(top, 0), min(bottom, h)        # numpy slicing clips (negative starts would wrap: not reached for centred fields)
        l, r = max(left, 0), min(right, w)
        self._strip_rows, self._strip_cols = (t, b), (l, r)
        xs = self._frame_sums(ctx, batch, (t, 0, b - t, w))[0] / (b - t)
        ys = self._frame_sums(ctx, batch, (0, l, h, r - l))[1] / (r - l)
        # the strips as drawn by the reference (2x the image extent along the profile) and the central ROI (:320-338)
        self.x_rect = Rectangle(width=w * 2, height=b - t, center=(x, y))
        self.y_rect = Rectangle(width=r - l, height=h * 2, center=(x, y))
        self.center_rect = RectangleROI(array=self._frame_u16(), width=right - left, height=bottom - top, center=Point(x, y))
        return xs, ys

    def _get_x_y_position(self, ctx, batch, position):
        """field_profile_analysis.py:343-368"""
        if self._centering != Centering.MANUAL:
            colsum, rowsum = self._frame_sums(ctx, batch)
            cls = PROFILES[self._edge_type]
            v_p = cls(values=colsum, dpmm=self.image.dpmm)
            h_p = cls(values=rowsum, dpmm=self.image.dpmm)
            if self._centering == Centering.BEAM_CENTER:
                return v_p.center_idx, h_p.center_idx
            return v_p.cax_index, h_p.cax_index
        if len(position) != 2:
            raise ValueError("Position must be a tuple of two values")
        if any(pos < 0 or pos > 1 for pos in position):
            raise ValueError("Position values must be between 0 and 1")
        return self.image.shape[1] * position[1], self.image.shape[0] * position[0]

    def _generate_results_data(self) -> FieldProfileResult:
        if not self._is_analyzed:
            raise NotAnalyzed("Image is not analyzed yet. Use analyze() first.")

        def pack(p):
            return {k: float(v) for k, v in p.metric_values.items()} | {"Field Width (mm)": p.field_width_mm, "values": p.values.tolist()}

        c = self.center_rect
        return FieldProfileResult(edge_type=self._edge_type.value, normalization=str(self._normalization.value),
                                  centering=self._centering.value, x_metrics=pack(self.x_profile), y_metrics=pack(self.y_profile),
                                  center={"mean": c.mean, "stdev": c.std, "min": c.min, "max": c.max})

    def results(self) -> str:
        """field_profile_analysis.py:221-233"""
        d = self.results_data(as_dict=True)
        s = ""
        for key, value in d.items():
            if isinstance(value, dict):
                s += f"{key}:\n"
                for k, v in value.items():
                    if not isinstance(v, list):
                        s += f"{k}: {v}\n"
            else:
                s += f"{key}: {value}\n"
        return s


def analyze_batch(frames, dpmm: float, *, device: int | None = None, sid: float = 1000.0, **analyze_kwargs) -> list[FieldProfileAnalysis]:
    """``FieldProfileAnalysis(frame, dpi=..., sid=...).analyze(**analyze_kwargs)`` for every frame of ``frames`` (uint16 [n, h, w]).

    The frames are uploaded once; histogram inversion check, field-centre sums, strip sums and central-ROI statistics of ALL frames
    come from batch launches (``epid_frame_stats`` with percentiles / views, ``epid_roi_stats``); only the profile / metric objects
    are per-frame Python (the plug-in contract).  Returns analysed ``FieldProfileAnalysis`` objects."""
    a = np.asarray(frames)
    if a.ndim == 2:
        a = a[None]
    if a.dtype != np.uint16:
        raise TypeError("field-profile frames must be uint16")
    ctx = nat.Context.default(device)
    out = []
    with nat.Batch.upload(ctx, a) as batch:
        stats = _BatchStats(ctx, batch)
        for i in range(len(a)):
            f = FieldProfileAnalysis.__new__(FieldProfileAnalysis)
            f.image = image.ArrayImage(a[i], dpi=dpmm * 25.4 * 1000.0 / sid, sid=sid)
            f._is_analyzed = False
            f._warnings = []
            f._flipped = stats.hist_inverted(i)  # check_inversion_by_histogram() of the constructor
            if f._flipped:
                f.image.invert()
            f._shared = (stats, i)
            f.analyze(**analyze_kwargs)
            del f._shared
            out.append(f)
    return out


class _BatchStats:
    """Whole-batch device statistics shared by the per-frame objects of ``analyze_batch``: one launch per distinct view."""

    def __init__(self, ctx, batch):
        self.ctx, self.batch = ctx, batch
        self.full = nat.frame_stats(ctx, batch, percentiles=(5, 50, 95))
        self.views = {}

    def hist_inverted(self, i: int) -> bool:      # core/image.py:899-926
        lo, mid, hi = self.full["percentiles"][i]
        return bool(abs(mid - lo) > abs(mid - hi))

    def view(self, view):
        if view not in self.views:
            self.views[view] = nat.frame_stats(self.ctx, self.batch, view=view)
        return self.views[view]
