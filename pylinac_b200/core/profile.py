"""1-D profile operators -- mirror of the parts of ``pylinac/core/profile.py`` the hot path uses.

All arithmetic on profile values runs in CUDA through the C-ABI (``epid_find_peaks`` and the element-wise / stencil operators of
``core.array_utils``); index bookkeeping stays in Python.  There is no numpy / scipy compute fallback.

    enums Interpolation / Normalization / Edge / Centering        core/profile.py:160-192
    find_peaks                                                    core/profile.py:2545-2649
    MultiProfile.find_peaks / find_valleys / find_fwxm_peaks      core/profile.py:2021-2176
    ProfileMixin (invert / normalize / stretch / ground / filter) core/profile.py:86-159
    FWXMProfile.field_edge_idx / center_idx / field_width_px      core/profile.py:322-344, 582-611
"""
from __future__ import annotations

import enum

import numpy as np

from .. import _native as nat
from . import array_utils as utils
from .geometry import Point


class Interpolation(enum.Enum):
    """core/profile.py:160-165"""

    NONE = None
    LINEAR = "Linear"
    SPLINE = "Spline"


class Normalization(enum.Enum):
    """core/profile.py:168-174"""

    NONE = None
    GEOMETRIC_CENTER = "Geometric center"
    BEAM_CENTER = "Beam center"
    MAX = "Max"


class Edge(enum.Enum):
    """core/profile.py:177-182"""

    FWHM = "FWHM"
    INFLECTION_DERIVATIVE = "Inflection Derivative"
    INFLECTION_HILL = "Inflection Hill"


class Centering(enum.Enum):
    """core/profile.py:185-190"""

    MANUAL = "Manual"
    BEAM_CENTER = "Beam center"
    GEOMETRIC_CENTER = "Geometric center"


def find_peaks(values, threshold=-np.inf, peak_separation=0, max_number=None, fwxm_height=0.5, min_width=0,
               search_region=(0.0, 1.0), peak_sort="prominences", required_prominence=None):
    """core/profile.py:2545-2623 -- scipy.signal.find_peaks semantics, executed by the CUDA kernel behind epid_find_peaks."""
    return nat.find_peaks(nat.Context.default(), np.asarray(values, dtype=np.float64), threshold=threshold,
                          peak_separation=peak_separation, max_number=max_number, fwxm_height=fwxm_height, min_width=min_width,
                          search_region=search_region, peak_sort=peak_sort, required_prominence=required_prominence)


class ProfileMixin:
    """core/profile.py:86-159: in-place value operators of 1-D profiles (device arithmetic via core.array_utils)."""

    values: np.ndarray

    def invert(self) -> None:
        self.values = utils.invert(self.values)

    def normalize(self, norm_val="max") -> None:
        self.values = utils.normalize(self.values, value=None if norm_val == "max" else norm_val)

    def stretch(self, min: float = 0, max: float = 1) -> None:
        self.values = utils.stretch(self.values, min=min, max=max)

    def ground(self) -> float:
        mn = float(np.asarray(self.values).min())
        self.values = utils.ground(self.values)
        return mn

    def filter(self, size: float = 0.05, kind: str = "median") -> None:
        self.values = utils.filter(self.values, size=size, kind=kind)


class MultiProfile(ProfileMixin):
    """core/profile.py:2002-2176"""

    def __init__(self, values):
        self.values = np.asarray(values)
        self.peaks: list[Point] = []
        self.valleys: list[Point] = []

    def find_peaks(self, threshold=0.3, min_distance=0.05, max_number=None, search_region=(0.0, 1.0), peak_sort="prominences"):
        idx, props = find_peaks(self.values, threshold=threshold, peak_separation=min_distance, max_number=max_number,
                                search_region=search_region, peak_sort=peak_sort)
        self.peaks = [Point(value=v, idx=i) for i, v in zip(idx, props["peak_heights"])]
        return idx, props["peak_heights"]

    def find_valleys(self, threshold=0.3, min_distance=0.05, max_number=None, search_region=(0.0, 1.0)):
        idx, props = find_peaks(utils_negate(self.values), threshold=threshold, peak_separation=min_distance, max_number=max_number,
                                search_region=search_region)
        vals = np.asarray(self.values)[idx]
        self.valleys = [Point(value=v, idx=i) for i, v in zip(idx, vals)]
        return idx, vals

    def find_fwxm_peaks(self, threshold=0.3, min_distance=0.05, max_number=None, search_region=(0.0, 1.0),
                        peak_sort="prominences", required_prominence=None):
        _, props = find_peaks(self.values, threshold=threshold, peak_separation=min_distance, max_number=max_number,
                              search_region=search_region, peak_sort=peak_sort, required_prominence=required_prominence)
        idxs = [int(round(lt + (rt - lt) / 2)) for lt, rt in zip(props["left_ips"], props["right_ips"])]
        vals = [np.asarray(self.values)[i] for i in idxs]
        self.peaks = [Point(value=v, idx=i) for i, v in zip(idxs, vals)]
        return np.array(idxs), np.array(vals)


class CircleProfile(MultiProfile):
    """core/profile.py:2179-2402: a profile sampled on a circle (nearest neighbour), peaks mapped back to image coordinates."""

    def __init__(self, center, radius: float, image_array: np.ndarray, start_angle: float = 0, ccw: bool = True,
                 sampling_ratio: float = 1.0):
        self.center = Point(center)
        self.radius = radius
        self.image_array = image_array
        self.start_angle = start_angle
        self.ccw = ccw
        self.sampling_ratio = sampling_ratio
        prof, self.x_locations, self.y_locations = self._sample()
        super().__init__(prof)

    def _sample(self):
        return nat.circle_profile(nat.Context.default(), self.image_array, (self.center.x, self.center.y), self.radius,
                                  start_angle=self.start_angle, ccw=self.ccw, sampling_ratio=self.sampling_ratio)

    @property
    def size(self) -> float:
        return np.pi * self.radius * 2 * self.sampling_ratio

    def _map_peaks(self) -> None:
        for peak in self.peaks:
            peak.x = self.x_locations[int(peak.idx)]
            peak.y = self.y_locations[int(peak.idx)]

    def find_peaks(self, threshold=0.3, min_distance=0.05, max_number=None, search_region=(0.0, 1.0)):
        out = super().find_peaks(threshold, min_distance, max_number, search_region)
        self._map_peaks()
        return out

    def find_valleys(self, threshold=0.3, min_distance=0.05, max_number=None, search_region=(0.0, 1.0)):
        out = super().find_valleys(threshold, min_distance, max_number, search_region)
        self._map_peaks()
        return out

    def find_fwxm_peaks(self, threshold=0.3, min_distance=0.05, max_number=None, search_region=(0.0, 1.0)):
        out = super().find_fwxm_peaks(threshold, min_distance, max_number, search_region=search_region)
        self._map_peaks()
        return out

    def roll(self, amount: int) -> None:
        self.values = np.roll(self.values, -amount)
        self.x_locations = np.roll(self.x_locations, -amount)
        self.y_locations = np.roll(self.y_locations, -amount)


class CollapsedCircleProfile(CircleProfile):
    """core/profile.py:2405-2483: mean of `num_profiles` circle profiles in a band of relative width `width_ratio`."""

    def __init__(self, center, radius: float, image_array: np.ndarray, start_angle: float = 0, ccw: bool = True,
                 sampling_ratio: float = 1.0, width_ratio: float = 0.1, num_profiles: int = 20):
        if not 0 <= width_ratio <= 1:
            raise ValueError("width_ratio must be between 0 and 1")
        self.width_ratio = width_ratio
        self.num_profiles = num_profiles
        super().__init__(center, radius, image_array, start_angle, ccw, sampling_ratio)

    def _sample(self):
        return nat.circle_profile(nat.Context.default(), self.image_array, (self.center.x, self.center.y), self.radius,
                                  start_angle=self.start_angle, ccw=self.ccw, sampling_ratio=self.sampling_ratio, collapsed=True,
                                  width_ratio=self.width_ratio, num_profiles=self.num_profiles)

    @property
    def size(self) -> float:
        return np.pi * self.radius * (1 + self.width_ratio) * 2 * self.sampling_ratio


_NORM_CODE = {Normalization.NONE: 0, Normalization.GEOMETRIC_CENTER: 1, Normalization.BEAM_CENTER: 2, Normalization.MAX: 3}


class SingleProfile(ProfileMixin):
    """core/profile.py:1119-1937 -- same constructor and query methods; the numerics (interpolation, grounding, normalisation,
    FWXM / inflection edges, penumbra, field data) are the device engine of csrc/field.cu behind ``epid_single_profile``.

    * Interpolation NONE / LINEAR over ``range(len(values))`` happens on the device.  Interpolation SPLINE (cubic ``interp1d``:
      not-a-knot spline) and custom ``x_values`` are resampled on the host onto the reference's ``linspace`` grid (one tridiagonal
      solve over the few hundred raw samples) and handed to the engine as a pre-sampled profile; custom ``x_values`` with
      interpolation NONE (possibly unevenly spaced, e.g. ion-chamber arrays) travel to the engine as explicit abscissae.
    * Edge.INFLECTION_HILL: the derivative edges come from the engine, the two 4-parameter Hill fits (a few dozen samples each,
      core/hill.py) run on the host, and the fitted inflection points go back to the engine as the field edges for everything
      downstream (beam centre, normalisation, field data)."""

    def __init__(self, values, dpmm: float | None = None, interpolation=Interpolation.LINEAR, ground: bool = True,
                 interpolation_resolution_mm: float = 0.1, interpolation_factor: float = 10,
                 normalization_method=Normalization.BEAM_CENTER, edge_detection_method=Edge.FWHM,
                 edge_smoothing_ratio: float = 0.003, hill_window_ratio: float = 0.1, x_values=None, centering=Centering.BEAM_CENTER):
        self._interp_method = interpolation if isinstance(interpolation, Interpolation) else Interpolation(interpolation)
        self._norm_method = normalization_method if isinstance(normalization_method, Normalization) else Normalization(normalization_method)
        self._edge_method = edge_detection_method if isinstance(edge_detection_method, Edge) else Edge(edge_detection_method)
        self._centering = centering if isinstance(centering, Centering) else Centering(centering)
        raw = np.asarray(values, dtype=np.float64)
        if raw.ndim != 1:
            raise ValueError("Profile values must be 1-D")
        self.dpmm = dpmm
        self._interpolation_res = interpolation_resolution_mm
        self._interpolation_factor = interpolation_factor
        self._ground = ground
        self._edge_smoothing_ratio = edge_smoothing_ratio
        self._hill_window_ratio = hill_window_ratio
        sp = nat.SpParams()
        sp.dpmm = float(dpmm) if dpmm else 0.0
        sp.interpolation = 0 if self._interp_method == Interpolation.NONE else 1
        sp.interpolation_resolution_mm = float(interpolation_resolution_mm)
        sp.interpolation_factor = float(interpolation_factor)
        custom_x = x_values is not None and not np.array_equal(np.asarray(x_values), np.arange(len(raw)))
        if custom_x or self._interp_method == Interpolation.SPLINE:
            raw, self._x_explicit = self._presample(raw, x_values)
            sp.interpolation, sp.x_start, sp.x_stop = 2, float(self._x_explicit[0]), float(self._x_explicit[-1])
        else:
            self._x_explicit = None
        self._raw = raw
        sp.ground = 1 if ground else 0
        sp.normalization = _NORM_CODE[self._norm_method]
        sp.edge = {Edge.FWHM: 0, Edge.INFLECTION_DERIVATIVE: 1, Edge.INFLECTION_HILL: 2}[self._edge_method]
        sp.centering = 2 if self._centering == Centering.GEOMETRIC_CENTER else 1
        sp.edge_smoothing_ratio = float(edge_smoothing_ratio)
        self._params = sp
        self._cache = {}
        if self._edge_method == Edge.INFLECTION_HILL:
            self._hill_first_pass()
        r, vals, _ = self._query()
        if int(r["status"]) != 0:
            raise IndexError("no peak was found in the profile")       # what find_peaks(...)[0] raises in the reference
        self.values = vals
        self.x_indices = self._x_explicit if self._x_explicit is not None else \
            np.linspace(float(r["x_start"]), float(r["x_stop"]), num=int(r["n"]))

    def gamma(self, evaluation_profile, distance_to_agreement: int = 1, dose_to_agreement: float = 1, gamma_cap_value: float = 2,
              dose_threshold: float = 5, global_dose: bool = True, fill_value: float = np.nan) -> np.ndarray:
        """core/profile.py:1939-1993: ``core.gamma.gamma_1d`` of the two profiles over their ``x_indices`` (note the argument order:
        distance first); both profiles need ``dpmm``."""
        from .gamma import gamma_1d

        if not self.dpmm or not evaluation_profile.dpmm:
            raise ValueError("At least one profile does not have the dpmm attribute. Physical spacing cannot be determined. Set it "
                             "before performing gamma analysis.")
        return gamma_1d(reference=self.values, evaluation=evaluation_profile.values, reference_coordinates=self.x_indices,
                        evaluation_coordinates=evaluation_profile.x_indices, dose_to_agreement=dose_to_agreement,
                        distance_to_agreement=distance_to_agreement, gamma_cap_value=gamma_cap_value, global_dose=global_dose,
                        dose_threshold=dose_threshold, fill_value=fill_value)[0]

    # -- _interpolate (core/profile.py:1306-1360) for the cases the device interpolation does not cover
    def _presample(self, raw: np.ndarray, x_values):
        x = np.arange(len(raw), dtype=np.float64) if x_values is None else np.asarray(x_values, dtype=np.float64)
        if len(x) != len(raw):
            raise ValueError("x_values and values must have the same length")
        if np.diff(x).min() < 0:
            raise ValueError("Profile values must be monotonically increasing")
        if self._interp_method == Interpolation.NONE:
            return raw, x
        samples = int(round(len(x) / (self.dpmm * self._interpolation_res))) if self.dpmm is not None \
            else int(round(len(x) * self._interpolation_factor))
        resampling_factor = samples / len(raw)
        offset = 0.5 - 1 / (2 * resampling_factor)
        new_x = np.linspace(x[0] - offset, x[-1] + offset, num=samples)
        if self._interp_method == Interpolation.LINEAR:
            new_y = _linear_spline(x, raw, new_x)            # interp1d(kind="linear", fill_value="extrapolate")
        else:
            new_y = _cubic_spline_eval(x, raw, _not_a_knot_cubic(x, raw), new_x)     # interp1d(kind="cubic", fill_value="extrapolate")
        return new_y, new_x

    # -- Edge.INFLECTION_HILL (core/profile.py:1678-1721)
    def _y_at(self, values: np.ndarray, x_grid: np.ndarray, q):
        return _linear_spline(x_grid, values, q)

    def _fit_hills(self, values: np.ndarray, x_grid: np.ndarray, left_idx: float, right_idx: float):
        from .hill import Hill

        half = int(round(self._hill_window_ratio * abs(right_idx - left_idx) / 2))
        xl = np.arange(left_idx - half, left_idx + half)
        xl = xl[xl >= 0]
        xr = np.arange(right_idx - half, right_idx + half)
        xr = xr[xr < len(values)]
        return Hill.fit(xl, self._y_at(values, x_grid, xl)), Hill.fit(xr, self._y_at(values, x_grid, xr))

    def _hill_first_pass(self) -> None:
        """Derivative edges and un-normalised values from the engine, Hill fits on the host, fitted inflection points -> engine."""
        import copy

        first = copy.copy(self._params)
        first.edge, first.normalization = 1, 0
        r, vals, _ = nat.single_profile(nat.Context.default(), self._raw, first, x_values=self._x_explicit)
        if int(r["status"]) != 0 or not r["infl_ok"]:
            raise IndexError("no inflection points were found")
        self._deriv_edges = (float(r["infl_left"]), float(r["infl_right"]))
        grid = self._x_explicit if self._x_explicit is not None else np.linspace(float(r["x_start"]), float(r["x_stop"]), num=int(r["n"]))
        lh, rh = self._fit_hills(vals, grid, *self._deriv_edges)
        self._params.edge_left = lh.inflection_idx()["index (exact)"]
        self._params.edge_right = rh.inflection_idx()["index (exact)"]

    def _hills(self):
        """The fits ``inflection_data()`` of the reference makes on the final (normalised) values."""
        if "hills" not in self._cache:
            self._cache["hills"] = self._fit_hills(self.values, self.x_indices, *self._deriv_edges)
        return self._cache["hills"]

    def resample(self, interpolation_factor: int = 10, interpolation_resolution_mm: float = 0.1) -> "SingleProfile":
        """core/profile.py:1283-1304"""
        return SingleProfile(values=self.values, x_values=self.x_indices, dpmm=1 / self._interpolation_res if self.dpmm else None,
                             interpolation=self._interp_method, ground=self._ground,
                             interpolation_resolution_mm=interpolation_resolution_mm, interpolation_factor=interpolation_factor,
                             normalization_method=self._norm_method, edge_detection_method=self._edge_method,
                             edge_smoothing_ratio=self._edge_smoothing_ratio, hill_window_ratio=self._hill_window_ratio)

    def _query(self, fwxm_x=50.0, penumbra=(20.0, 80.0), in_field_ratio=0.8, slope_exclusion_ratio=0.2):
        key = (float(fwxm_x), float(penumbra[0]), float(penumbra[1]), float(in_field_ratio), float(slope_exclusion_ratio))
        if key not in self._cache:
            self._cache[key] = nat.single_profile(nat.Context.default(), self._raw, self._params, fwxm_x=fwxm_x, penumbra=penumbra,
                                                  in_field_ratio=in_field_ratio, slope_exclusion_ratio=slope_exclusion_ratio,
                                                  x_values=self._x_explicit)
        return self._cache[key]

    # -- core/profile.py:1373-1409
    def geometric_center(self) -> dict:
        r, _, _ = self._query()
        return {"index (exact)": float(r["geometric_center_index"]), "value (exact)": float(r["geometric_center_value"])}

    def beam_center(self) -> dict:
        r, _, _ = self._query()
        if not r["beam_ok"]:
            raise IndexError("no field edges were found")
        idx = float(r["beam_center_index"])
        return {"index (rounded)": int(round(idx)), "index (exact)": idx, "value (@rounded)": float(r["beam_center_value_at_rounded"])}

    # -- core/profile.py:1411-1461
    def fwxm_data(self, x: float = 50) -> dict:
        if not 0 <= x <= 100:
            raise ValueError("x must be between 0 and 100")
        r, _, _ = self._query(fwxm_x=x)
        if not r["fwxm_ok"]:
            raise IndexError("no peak was found in the profile")
        left, right = float(r["fwxm_left"]), float(r["fwxm_right"])
        width = right - left
        center = (right - left) / 2 + left
        data = {"width (exact)": width, "width (rounded)": int(round(width)), "center index (rounded)": int(round(center)),
                "center index (exact)": center, "center value (@rounded)": float(r["fwxm_center_value_at_rounded"]),
                "left index (exact)": left, "left index (rounded)": int(round(left)),
                "left value (@rounded)": float(r["fwxm_left_value_at_rounded"]), "right index (exact)": right,
                "right index (rounded)": int(round(right)), "right value (@rounded)": float(r["fwxm_right_value_at_rounded"])}
        if self.dpmm:
            data["width (exact) mm"] = width / self.dpmm
            data["left distance (exact) mm"] = abs(center - left) / self.dpmm
            data["right distance (exact) mm"] = abs(right - center) / self.dpmm
        return data

    # -- core/profile.py:1635-1721
    def inflection_data(self) -> dict:
        if self._edge_method == Edge.FWHM:
            raise ValueError("FWHM edge method does not have inflection points. Use a different edge detection method")
        if self._edge_method == Edge.INFLECTION_HILL:
            lh, rh = self._hills()
            li, ri = lh.inflection_idx(), rh.inflection_idx()
            return {"left index (rounded)": li["index (rounded)"], "left index (exact)": li["index (exact)"],
                    "right index (rounded)": ri["index (rounded)"], "right index (exact)": ri["index (exact)"],
                    "left value (@exact)": lh.y(li["index (exact)"]), "right value (@exact)": rh.y(ri["index (exact)"]),
                    "left Hill params": lh.params, "right Hill params": rh.params}
        r, _, _ = self._query()
        if not r["infl_ok"]:
            raise IndexError("no inflection points were found")
        left, right = float(r["infl_left"]), float(r["infl_right"])
        return {"left index (rounded)": int(round(left)), "left index (exact)": left, "right index (rounded)": int(round(right)),
                "right index (exact)": right, "left value (@rounded)": float(r["infl_left_value_rounded"]),
                "left value (@exact)": float(r["infl_left_value_exact"]), "right value (@rounded)": float(r["infl_right_value_rounded"]),
                "right value (@exact)": float(r["infl_right_value_exact"])}

    # -- core/profile.py:1723-1907
    def penumbra(self, lower: int = 20, upper: int = 80) -> dict:
        if lower > upper:
            raise ValueError("Upper penumbra value must be larger than the lower penumbra value")
        if self._edge_method == Edge.INFLECTION_HILL:
            return self._hill_penumbra(lower, upper)
        r, _, _ = self._query(penumbra=(lower, upper))
        if not r["pen_ok"]:
            raise IndexError("no field edges were found")
        data = {f"left {lower}% index (exact)": float(r["pen_left_lower"]), f"left {upper}% index (exact)": float(r["pen_left_upper"]),
                f"right {lower}% index (exact)": float(r["pen_right_lower"]), f"right {upper}% index (exact)": float(r["pen_right_upper"]),
                "left penumbra width (exact)": abs(float(r["pen_left_upper"]) - float(r["pen_left_lower"])),
                "right penumbra width (exact)": abs(float(r["pen_right_upper"]) - float(r["pen_right_lower"]))}
        if self.dpmm:
            data["left penumbra width (exact) mm"] = data["left penumbra width (exact)"] / self.dpmm
            data["right penumbra width (exact) mm"] = data["right penumbra width (exact)"] / self.dpmm
        return data

    def _hill_penumbra(self, lower, upper) -> dict:
        """core/profile.py:1853-1907: positions where the fitted Hill curves reach lower / 50 and upper / 50 of their inflection
        values"""
        infl = self.inflection_data()
        lh, rh = self._hills()
        ll_v, ul_v = infl["left value (@exact)"] * lower / 50, infl["left value (@exact)"] * upper / 50
        lr_v, ur_v = infl["right value (@exact)"] * lower / 50, infl["right value (@exact)"] * upper / 50
        ll, ul, lr, ur = lh.x(ll_v), lh.x(ul_v), rh.x(lr_v), rh.x(ur_v)
        data = {f"left {lower}% index (exact)": ll, f"left {lower}% value (exact)": ll_v, f"left {upper}% index (exact)": ul,
                f"left {upper}% value (exact)": ul_v, f"right {lower}% index (exact)": lr, f"right {lower}% value (exact)": lr_v,
                f"right {upper}% index (exact)": ur, f"right {upper}% value (exact)": ur_v,
                "left values": self.values[int(round(ll)):int(round(ul))], "right values": self.values[int(round(ur)):int(round(lr))],
                "left penumbra width (exact)": abs(ul - ll), "right penumbra width (exact)": abs(ur - lr),
                "left gradient (exact)": lh.gradient_at(infl["left index (exact)"]),
                "right gradient (exact)": rh.gradient_at(infl["right index (exact)"])}
        if self.dpmm:
            data["left penumbra width (exact) mm"] = data["left penumbra width (exact)"] / self.dpmm
            data["left gradient (exact) %/mm"] = data["left gradient (exact)"] * self.dpmm * 100
            data["right penumbra width (exact) mm"] = data["right penumbra width (exact)"] / self.dpmm
            data["right gradient (exact) %/mm"] = data["right gradient (exact)"] * self.dpmm * 100
        return data

    # -- core/profile.py:1463-1633
    def field_data(self, in_field_ratio: float = 0.8, slope_exclusion_ratio: float = 0.2) -> dict:
        if slope_exclusion_ratio >= in_field_ratio:
            raise ValueError("The exclusion region must be smaller than the field ratio")
        r, _, fv = self._query(in_field_ratio=in_field_ratio, slope_exclusion_ratio=slope_exclusion_ratio)
        if not r["fd_ok"]:
            raise IndexError("no field edges were found")
        g = lambda k: float(r[k])
        data = {"width (exact)": g("fd_width"), "beam center index (exact)": g("fd_beam_center"),
                "beam center index (rounded)": int(round(g("fd_beam_center"))), "beam center value (@rounded)": g("fd_beam_center_value"),
                "cax index (exact)": g("fd_cax"), "cax index (rounded)": int(round(g("fd_cax"))), "cax value (@rounded)": g("fd_cax_value"),
                "left index (exact)": g("fd_left"), "left index (rounded)": int(round(g("fd_left"))), "left value (@rounded)": g("fd_left_value"),
                "left slope": g("fd_left_slope"), "left intercept": g("fd_left_intercept"), "right slope": g("fd_right_slope"),
                "right intercept": g("fd_right_intercept"), "left inner index (exact)": g("fd_inner_left"),
                "left inner index (rounded)": int(round(g("fd_inner_left"))), "right inner index (exact)": g("fd_inner_right"),
                "right inner index (rounded)": int(round(g("fd_inner_right"))), '"top" index (exact)': g("fd_top_index"),
                '"top" index (rounded)': int(round(g("fd_top_index"))), '"top" value (@exact)': g("fd_top_value"),
                "top params": np.array(r["fd_top_params"], dtype=float), "right index (exact)": g("fd_right"),
                "right index (rounded)": int(round(g("fd_right"))), "right value (@rounded)": g("fd_right_value"), "field values": fv}
        if self.dpmm:
            d = self.dpmm
            data["width (exact) mm"] = data["width (exact)"] / d
            data["left slope (%/mm)"] = data["left slope"] * d * 100
            data["right slope (%/mm)"] = data["right slope"] * d * 100
            data["left distance->beam center (exact) mm"] = abs(data["beam center index (exact)"] - data["left index (exact)"]) / d
            data["right distance->beam center (exact) mm"] = abs(data["right index (exact)"] - data["beam center index (exact)"]) / d
            data["left distance->CAX (exact) mm"] = abs(data["cax index (exact)"] - data["left index (exact)"]) / d
            data["right distance->CAX (exact) mm"] = abs(data["cax index (exact)"] - data["right index (exact)"]) / d
            data["left distance->top (exact) mm"] = abs(data['"top" index (exact)'] - data["left index (exact)"]) / d
            data["right distance->top (exact) mm"] = abs(data['"top" index (exact)'] - data["right index (exact)"]) / d
            data['"top"->beam center (exact) mm'] = (data['"top" index (exact)'] - data["beam center index (exact)"]) / d
            data['"top"->CAX (exact) mm'] = abs(data['"top" index (exact)'] - data["cax index (exact)"]) / d
        return data

    # -- core/profile.py:1909-1937
    def field_calculation(self, in_field_ratio: float = 0.8, calculation: str = "mean", slope_exclusion_ratio: float = 0.2):
        if calculation not in ("mean", "median", "max", "min", "area"):
            raise ValueError("calculation must be one of mean, median, max, min, area")
        fv = self.field_data(in_field_ratio, slope_exclusion_ratio=slope_exclusion_ratio)["field values"]
        if calculation == "max":
            return float(fv.max())
        if calculation == "min":
            return float(fv.min())
        srt = np.sort(fv)                     # a few hundred field values: selection / pairwise sum on the host-resident result
        if calculation == "median":
            m = len(srt)
            return float(srt[m // 2] if m % 2 else (srt[m // 2 - 1] + srt[m // 2]) / 2)
        if calculation == "mean":
            return float(fv.mean())
        return None


def utils_negate(values) -> np.ndarray:
    """-values for find_valleys: a sign flip of the stored samples (no arithmetic on magnitudes)."""
    return np.negative(np.asarray(values, dtype=np.float64))


def _linear_spline(xk: np.ndarray, yk: np.ndarray, xq):
    """UnivariateSpline(x, y, k=1, s=0)(xq) (core/profile.py:249-274): the interpolating linear B-spline, evaluated like FITPACK's
    splev -- y0 * (x1 - x) / (x1 - x0) + y1 * (x - x0) / (x1 - x0) on the knot interval that holds x (extrapolating the end
    intervals)."""
    xq_arr = np.atleast_1d(np.asarray(xq, dtype=np.float64))
    i = np.clip(np.searchsorted(xk, xq_arr, side="right") - 1, 0, len(xk) - 2)
    x0, x1 = xk[i], xk[i + 1]
    d = x1 - x0
    out = yk[i] * ((x1 - xq_arr) / d) + yk[i + 1] * ((xq_arr - x0) / d)
    return float(out[0]) if np.ndim(xq) == 0 else out


def _interp1d_linear(xs: np.ndarray, ys: np.ndarray, xq: float) -> float:
    """scipy interp1d(x, y) (kind linear, assume_sorted False) at one point: stable sort by x, then _call_linear
    (scipy/interpolate/_interpolate.py): slope * (x_new - x_lo) + y_lo on the bracketing samples; out of range raises."""
    order = np.argsort(xs, kind="mergesort")
    x, y = xs[order], ys[order]
    if xq < x[0] or xq > x[-1]:
        raise ValueError("A value in x_new is outside the interpolation range.")
    hi = int(np.clip(np.searchsorted(x, xq), 1, len(x) - 1))
    lo = hi - 1
    slope = (y[hi] - y[lo]) / (x[hi] - x[lo])
    return float(slope * (xq - x[lo]) + y[lo])


class ProfileBase(ProfileMixin):
    """core/profile.py:195-575: a single-field profile with linear look-ups between samples, in-field extraction and metric
    plug-ins.  ``field_edge_idx`` comes from the subclass; the peak search behind it runs on the GPU (``find_peaks``)."""

    def __init__(self, values, x_values=None, ground: bool = False, normalization=Normalization.NONE):
        values = np.asarray(values, dtype=np.float64)
        if values.ndim != 1:
            raise ValueError("Profile values must be 1-D")
        self.metrics = []
        self.metric_values = {}
        if x_values is None:
            x_values = np.arange(len(values))
        x_values = np.asarray(x_values)
        xd = np.diff(x_values)
        if xd.max() > 0 > xd.min():
            raise ValueError("X values must be monotonically increasing or decreasing")
        order = np.argsort(x_values)
        self.x_values = x_values[order]
        self.values = values[order]
        self._cache = {}
        if ground:
            self.values = utils.ground(self.values)
        # as in the reference the argument is compared with the enum MEMBERS: a plain string ("Max") selects no normalisation
        # (FieldProfileAnalysis hands the caller's raw argument through, field_profile_analysis.py:176-181)
        norm = normalization
        if norm == Normalization.MAX:
            self.values = utils.normalize(self.values)
        elif norm == Normalization.GEOMETRIC_CENTER:
            self.values = utils.normalize(self.values, utils.geometric_center_value(self.values))
        elif norm == Normalization.BEAM_CENTER:
            self.values = utils.normalize(self.values, self.y_at_x(self.center_idx))
            self._cache = {}

    # -- look-ups (core/profile.py:249-288)
    def x_at_x_idx(self, x):
        return _linear_spline(np.arange(len(self.x_values), dtype=np.float64), self.x_values.astype(np.float64), x)

    def x_idx_at_x(self, x: float) -> int:
        return int(np.argmin(np.abs(self.x_values - x)))

    def y_at_x(self, x):
        return _linear_spline(self.x_values.astype(np.float64), self.values, x)

    def x_at_y(self, y: float, side: str) -> float:
        s = self.x_idx_at_x(self.center_idx)
        if side == "left":
            return _interp1d_linear(self.values[:s], self.x_values[:s].astype(np.float64), float(y))
        return _interp1d_linear(self.values[s:], self.x_values[s:].astype(np.float64), float(y))

    def field_edge_idx(self, side: str) -> float:
        raise NotImplementedError

    def _edges(self):
        if "edges" not in self._cache:
            self._cache["edges"] = (self.field_edge_idx("left"), self.field_edge_idx("right"))
        return self._cache["edges"]

    # -- field geometry (core/profile.py:295-344)
    @property
    def center_idx(self) -> float:
        left, right = self._edges()
        return abs(right - left) / 2 + left

    @property
    def geometric_center_idx(self) -> float:
        return self.x_at_x_idx(utils.geometric_center_idx(self.values))

    @property
    def cax_index(self) -> float:
        return self.x_at_x_idx((len(self.x_values) - 1) / 2)

    @property
    def field_width_px(self) -> float:
        left, right = self._edges()
        return max(right, left) - min(right, left)

    def field_x_values(self, in_field_ratio: float) -> np.ndarray:
        import math

        left, right = self._edges()
        width = self.field_width_px
        f_left = left + (1 - in_field_ratio) / 2 * width
        f_right = right - (1 - in_field_ratio) / 2 * width
        lower, upper = math.floor(min(f_left, f_right)), math.ceil(max(f_left, f_right))
        return self.x_values[np.nonzero((self.x_values >= lower) & (self.x_values <= upper))[0]]

    def field_indices(self, in_field_ratio: float):
        xs = self.field_x_values(in_field_ratio)
        left, right = xs[0], xs[-1]
        return left, right, max(right, left) - min(right, left)

    def field_values(self, in_field_ratio: float = 0.8) -> np.ndarray:
        return self.y_at_x(self.field_x_values(in_field_ratio))

    # -- resampling (core/profile.py:355-437)
    def _resample_kwargs(self) -> dict:
        """The constructor arguments a resampled copy keeps (the per-class ``as_resampled`` overrides of the reference)."""
        return {}

    def _warn_small_int_range(self) -> None:
        arr_range = self.values.max() - self.values.min()
        if self.values.dtype != float and arr_range < 100:
            import warnings

            warnings.warn(f"Array range is small ({arr_range}) and is not a float. Interpolation may look step-like. "
                          "Consider converting the array to a float before passing it to this method.", UserWarning)

    def as_resampled(self, interpolation_factor: float = 10, order: int = 3):
        """A new profile of the same class ``interpolation_factor`` times denser: spline zoom of the values on the device
        (scipy.ndimage.zoom(order, mode='nearest', grid_mode=False) semantics, csrc/zoom.cu), x values spread linearly over the
        same extent."""
        self._warn_small_int_range()
        new_y = utils.zoom(self.values, interpolation_factor, order=order, mode="nearest")
        new_x = np.linspace(self.x_values.min(), self.x_values.max(), len(new_y))
        return type(self)(values=new_y, x_values=new_x, ground=False, normalization=Normalization.NONE, **self._resample_kwargs())

    def resample_to(self, target_profile):
        """The values of THIS profile linearly interpolated at the x positions of ``target_profile`` (physical positions for
        physical profiles); no extrapolation.  Returns a non-physical profile of this profile's class."""
        target_x = target_profile.physical_x_values if isinstance(target_profile, PhysicalProfileMixin) else target_profile.x_values
        self_x = self.physical_x_values if isinstance(self, PhysicalProfileMixin) else self.x_values
        target_x = np.asarray(target_x, dtype=np.float64)
        self_x = np.asarray(self_x, dtype=np.float64)
        if target_x.min() < self_x.min() or target_x.max() > self_x.max():
            raise ValueError("The target profile x-values are outside this profiles range. Extrapolation is not allowed. "
                             f"self x-values: {self_x.min()} to {self_x.max()}. target x-values: {target_x.min()} to {target_x.max()}. ")
        target_y = _linear_spline(self_x, self.values, target_x)
        output_type = type(self).__bases__[-1] if isinstance(self, PhysicalProfileMixin) else type(self)
        return output_type(values=target_y, x_values=target_x)

    # -- metric plug-ins (core/profile.py:541-575)
    def compute(self, metrics):
        from ..metrics.profile import ProfileMetric

        values = {}
        if isinstance(metrics, ProfileMetric):
            metrics = [metrics]
        key = None
        for metric in metrics:
            metric.inject_profile(self)
            self.metrics.append(metric)
            key, k = metric.full_name, 1
            while key in values or key in self.metric_values:      # uniquify
                key = f"{metric.full_name}-{k}"
                k += 1
            values[key] = metric.calculate()
        self.metric_values |= values
        return values[key] if len(values) == 1 else values

    def __len__(self):
        return len(self.values)


class FWXMProfile(ProfileBase):
    """core/profile.py:578-611: field edges = left / right interpolated positions of the largest peak at ``fwxm_height`` %."""

    def __init__(self, values, x_values=None, ground: bool = False, normalization=Normalization.NONE, fwxm_height: float = 50):
        self.fwxm_height = fwxm_height
        super().__init__(values, x_values=x_values, ground=ground, normalization=normalization)

    def _resample_kwargs(self) -> dict:
        return {"fwxm_height": self.fwxm_height}

    def field_edge_idx(self, side: str) -> float:
        _, props = find_peaks(self.values, fwxm_height=self.fwxm_height / 100, max_number=1)
        return float(self.x_at_x_idx(float(props["left_ips"][0] if side == "left" else props["right_ips"][0])))


def _not_a_knot_cubic(x: np.ndarray, y: np.ndarray):
    """Second derivatives M of the cubic spline through (x, y) with not-a-knot end conditions -- the interpolant of
    scipy interp1d(kind="cubic") (make_interp_spline(k=3), default boundary).  The two end conditions express M[0] and M[n-1]
    through their neighbours, which leaves a diagonally dominant tridiagonal system for M[1..n-2] (Thomas algorithm, O(n))."""
    n = len(x)
    h = np.diff(x).astype(np.float64)
    r = np.zeros(n)
    r[1:-1] = 6 * ((y[2:] - y[1:-1]) / h[1:] - (y[1:-1] - y[:-2]) / h[:-1])
    lo = np.zeros(n)          # sub-diagonal, diagonal, super-diagonal of rows 1 .. n-2
    di = np.zeros(n)
    up = np.zeros(n)
    lo[2:-1] = h[1:-1]
    di[1:-1] = 2 * (h[:-1] + h[1:])
    up[1:-2] = h[1:-1]
    # not-a-knot at the left:  M0 = ((h0 + h1) M1 - h0 M2) / h1;  at the right:  M[n-1] = ((hl + hk) M[n-2] - hl M[n-3]) / hk
    h0, h1, hk, hl = h[0], h[1], h[-2], h[-1]
    di[1] += h0 * (h0 + h1) / h1
    up[1] = h1 - h0 * h0 / h1
    di[n - 2] += hl * (hl + hk) / hk
    lo[n - 2] = hk - hl * hl / hk
    M = np.zeros(n)
    cp = np.zeros(n)
    dp = np.zeros(n)
    cp[1] = up[1] / di[1]
    dp[1] = r[1] / di[1]
    for i in range(2, n - 1):
        den = di[i] - lo[i] * cp[i - 1]
        cp[i] = up[i] / den
        dp[i] = (r[i] - lo[i] * dp[i - 1]) / den
    M[n - 2] = dp[n - 2]
    for i in range(n - 3, 0, -1):
        M[i] = dp[i] - cp[i] * M[i + 1]
    M[0] = ((h0 + h1) * M[1] - h0 * M[2]) / h1
    M[n - 1] = ((hl + hk) * M[n - 2] - hl * M[n - 3]) / hk
    return M


def _cubic_spline_eval(x: np.ndarray, y: np.ndarray, M: np.ndarray, xq) -> np.ndarray:
    """The cubic spline with knot second derivatives M at xq; outside [x[0], x[-1]] the first / last polynomial piece continues
    (interp1d(fill_value="extrapolate") on a BSpline)."""
    xq = np.asarray(xq, dtype=np.float64)
    i = np.clip(np.searchsorted(x, xq, side="right") - 1, 0, len(x) - 2)
    h = x[i + 1] - x[i]
    t = xq - x[i]
    b = (y[i + 1] - y[i]) / h - h * (2 * M[i] + M[i + 1]) / 6
    return y[i] + t * (b + t * (M[i] / 2 + t * (M[i + 1] - M[i]) / (6 * h)))


def _cubic_stationary_near(x: np.ndarray, y: np.ndarray, M: np.ndarray, i0: int, want_max: bool) -> float:
    """Local extremum of the cubic spline nearest to sample i0 (where minimize(..., x0=x[i0]) of the reference ends up):
    roots of the quadratic derivative on the intervals around i0."""
    best, best_d = float(x[i0]), np.inf
    for i in range(max(i0 - 2, 0), min(i0 + 2, len(x) - 1)):
        h = x[i + 1] - x[i]
        # S(t) on [x_i, x_i+1], t = x - x_i:  S = y_i + b t + (M_i / 2) t^2 + ((M_i+1 - M_i) / (6 h)) t^3
        b = (y[i + 1] - y[i]) / h - h * (2 * M[i] + M[i + 1]) / 6
        c2, c3 = M[i] / 2, (M[i + 1] - M[i]) / (6 * h)
        roots = np.roots([3 * c3, 2 * c2, b]) if c3 != 0 else (np.array([-b / (2 * c2)]) if c2 != 0 else np.array([]))
        for t in roots:
            if abs(t.imag) > 0:
                continue
            t = float(t.real)
            if -1e-12 <= t <= h + 1e-12:
                curv = 2 * c2 + 6 * c3 * t
                if (curv < 0) == want_max and abs(x[i] + t - x[i0]) < best_d:
                    best, best_d = float(x[i] + t), abs(x[i] + t - x[i0])
    return best


class InflectionDerivativeProfile(ProfileBase):
    """core/profile.py:629-684: field edges = extrema of the cubic interpolant of the gradient of the gaussian-smoothed profile.
    The reference finds them with scipy.optimize.minimize started at the arg-max / arg-min sample; here the stationary point of
    the same not-a-knot cubic spline next to that sample is computed in closed form (agreement ~1e-6 samples, the BFGS
    tolerance).  The gaussian smoothing runs on the GPU."""

    def __init__(self, values, x_values=None, ground: bool = False, normalization=Normalization.NONE,
                 edge_smoothing_ratio: float = 0.003):
        self.edge_smoothing_ratio = edge_smoothing_ratio
        super().__init__(values, x_values=x_values, ground=ground, normalization=normalization)

    def _resample_kwargs(self) -> dict:
        return {"edge_smoothing_ratio": self.edge_smoothing_ratio}

    def _derivative(self):
        if "diff" not in self._cache:
            filtered = utils.gaussian_filter(self.values, self.edge_smoothing_ratio * len(self.values))
            diff = np.gradient(filtered)
            xs = self.x_values.astype(np.float64)
            self._cache["diff"] = (diff, _not_a_knot_cubic(xs, diff))
        return self._cache["diff"]

    def field_edge_idx(self, side: str) -> float:
        diff, M = self._derivative()
        xs = self.x_values.astype(np.float64)
        if side == "left":
            return _cubic_stationary_near(xs, diff, M, int(np.argmax(diff)), want_max=True)
        return _cubic_stationary_near(xs, diff, M, int(np.argmin(diff)), want_max=False)


class HillProfile(InflectionDerivativeProfile):
    """core/profile.py:682-740: field edges = inflection points of Hill functions fitted to the penumbrae, each over a window
    of +/- ``hill_window_ratio`` x (distance between the two derivative edges) around its derivative edge."""

    def __init__(self, values, x_values=None, ground: bool = False, normalization=Normalization.NONE,
                 edge_smoothing_ratio: float = 0.003, hill_window_ratio: float = 0.1):
        self.hill_window_ratio = hill_window_ratio
        super().__init__(values, x_values=x_values, ground=ground, normalization=normalization,
                         edge_smoothing_ratio=edge_smoothing_ratio)

    def _resample_kwargs(self) -> dict:
        return {"edge_smoothing_ratio": self.edge_smoothing_ratio, "hill_window_ratio": self.hill_window_ratio}

    def field_edge_idx(self, side: str) -> float:
        from .hill import Hill

        left_infl = InflectionDerivativeProfile.field_edge_idx(self, "left")
        right_infl = InflectionDerivativeProfile.field_edge_idx(self, "right")
        window = (right_infl - left_infl) * self.hill_window_ratio
        centre = left_infl if side == "left" else right_infl
        lo, hi = self.x_idx_at_x(centre - window), self.x_idx_at_x(centre + window)
        fit = Hill.fit(self.x_values[lo:hi + 1], self.values[lo:hi + 1])
        return fit.inflection_idx()["index (exact)"]


class PhysicalProfileMixin:
    """core/profile.py:742-790"""

    def _init_physical(self, dpmm):
        self.dpmm = dpmm
        self.implicit_dpmm = float(np.mean(np.diff(self.x_values))) if dpmm is None else dpmm

    @property
    def physical_x_values(self) -> np.ndarray:
        if self.dpmm is None:
            return self.x_values
        return self.x_values / self.dpmm + 0.5 / self.dpmm

    @property
    def field_width_mm(self) -> float:
        return self.field_width_px / self.implicit_dpmm

    def as_simple_profile(self):
        """core/profile.py:932-949: the non-physical parent class over the physical x positions"""
        return type(self).__bases__[-1](values=self.values, x_values=self.physical_x_values)

    def gamma(self, evaluation_profile, dose_to_agreement: float = 3, distance_to_agreement: float = 3, gamma_cap_value: float = 2,
              dose_threshold: float = 5, fill_value: float = np.nan, return_profiles: bool = False):
        """core/profile.py:822-874: ``core.gamma.gamma_geometric`` of copies of both profiles, each shifted so that its geometric
        centre is at x = 0, over their physical x values.  ``return_profiles=True`` returns ``(gamma, reference, evaluation)`` with
        those copies."""
        import copy

        from .gamma import gamma_geometric

        if not isinstance(evaluation_profile, PhysicalProfileMixin):
            raise ValueError("The evaluation profile must also be a physical profile.")
        reference, evaluation = copy.deepcopy(self), copy.deepcopy(evaluation_profile)
        reference.x_values = reference.x_values - reference.geometric_center_idx
        evaluation.x_values = evaluation.x_values - evaluation.geometric_center_idx
        gamma = gamma_geometric(reference=reference.values, reference_coordinates=reference.physical_x_values,
                                evaluation=evaluation.values, evaluation_coordinates=evaluation.physical_x_values,
                                dose_to_agreement=dose_to_agreement, distance_to_agreement=distance_to_agreement,
                                gamma_cap_value=gamma_cap_value, dose_threshold=dose_threshold, fill_value=fill_value)
        return (gamma, reference, evaluation) if return_profiles else gamma

    def as_resampled(self, interpolation_resolution_mm: float = 0.1, order: int = 3, grid: bool = True):
        """core/profile.py:951-1013: resample to ``interpolation_resolution_mm`` per sample.  ``grid`` treats samples as pixels of
        physical size (scipy zoom grid_mode): the new x values then start / end half an (old minus new) pixel outside the old
        ones."""
        self._warn_small_int_range()
        factor = 1 / (self.dpmm * interpolation_resolution_mm)
        new_y = utils.zoom(self.values, factor, order=order, mode="nearest", grid_mode=grid)
        offset = 0.5 - 1 / (2 * factor) if grid else 0.0
        new_x = np.linspace(self.x_values.min() - offset, self.x_values.max() + offset, len(new_y))
        return type(self)(values=new_y, x_values=new_x, ground=False, normalization=Normalization.NONE, dpmm=factor * self.dpmm)


class FWXMProfilePhysical(PhysicalProfileMixin, FWXMProfile):
    """core/profile.py:1016-1047"""

    def __init__(self, values, dpmm: float | None = None, x_values=None, ground: bool = False, normalization=Normalization.NONE,
                 fwxm_height: float = 50):
        FWXMProfile.__init__(self, values, x_values=x_values, ground=ground, normalization=normalization, fwxm_height=fwxm_height)
        self._init_physical(dpmm)


class InflectionDerivativeProfilePhysical(PhysicalProfileMixin, InflectionDerivativeProfile):
    """core/profile.py:1050-1083"""

    def __init__(self, values, dpmm: float | None = None, x_values=None, ground: bool = False, normalization=Normalization.NONE,
                 edge_smoothing_ratio: float = 0.003):
        InflectionDerivativeProfile.__init__(self, values, x_values=x_values, ground=ground, normalization=normalization,
                                             edge_smoothing_ratio=edge_smoothing_ratio)
        self._init_physical(dpmm)


class HillProfilePhysical(PhysicalProfileMixin, HillProfile):
    """core/profile.py:1084-1116"""

    def __init__(self, values, dpmm: float | None = None, x_values=None, ground: bool = False, normalization=Normalization.NONE,
                 edge_smoothing_ratio: float = 0.003, hill_window_ratio: float = 0.1):
        HillProfile.__init__(self, values, x_values=x_values, ground=ground, normalization=normalization,
                             edge_smoothing_ratio=edge_smoothing_ratio, hill_window_ratio=hill_window_ratio)
        self._init_physical(dpmm)
