"""pylinac.ct's CatPhanBase (ct.py:321-534, 2027-2584, 3315-3401): the series, its localization, the air-bubble roll and the disk-ROI
modules, as far as the cheese phantoms and the ACR CT phantom use them.

One ``epid_ct_localize`` call (csrc/ct.cu) finds the phantom outline in every slice of the series: Slice.phantom_roi's Scharr edges,
Gaussian smoothing, Otsu threshold, clear_border, binary_fill_holes, labelling and region choice, bit-identical to the reference, on
either branch of get_regions (``clip_in_localization``: the clipped ndarray; otherwise the Slice, whose Otsu threshold is taken over a
110 mm disk around the image centre and scaled by 0.8).  ``find_phantom_axis`` (every slice) and ``find_origin_slice`` (every other
slice) both read its rows, where the reference runs the per-slice pipeline twice.  The roll's ``get_regions(slice)`` is one
``epid_ct_regions`` call: the region table with exact moments and each region's filled area; eccentricity follows on the host.  The
axis fit, the circle-profile percentiles, the origin choice and the roll are the reference's own numpy calls on the host; the circle
profiles and the disk ROI statistics run on the device (core.profile, core.roi).
"""
from __future__ import annotations

import os.path as osp
import warnings
from collections.abc import Callable
from fractions import Fraction
from pathlib import Path

import numpy as np
from pydantic import BaseModel

from . import _native as nat
from .core.geometry import Point
from .core.image import DicomImageStack
from .core.profile import CollapsedCircleProfile
from .core.roi import DiskROI, fill_disk_stats

# get_regions' Otsu disk on the Slice branch (ct.py:3334), in mm
OTSU_DISK_RADIUS_MM = 110


def z_position(metadata) -> float:
    """core/image.py:2378-2383: the slice's z, ImagePositionPatient[-1], else SliceLocation."""
    try:
        return metadata.ImagePositionPatient[-1]
    except AttributeError:
        return metadata.SliceLocation


class Region:
    """One row of get_regions(slice)'s region table (epid_ct_regions), with the regionprops attributes CatPhanBase's roll reads."""

    def __init__(self, row):
        self.label = int(row["label"])
        self.area = int(row["area"])
        self.filled_area = self.area_filled = int(row["filled_area"])
        self.bbox = tuple(int(v) for v in row["bbox"])
        self.bbox_area = self.area_bbox = (self.bbox[2] - self.bbox[0]) * (self.bbox[3] - self.bbox[1])
        # coords.mean(axis=0): the exact integer sums divided by the area
        self.centroid = (float(row["sum_r"]) / self.area, float(row["sum_c"]) / self.area)
        # central second moments from the exact sums about the bbox corner, as exact fractions
        n = self.area
        sr = int(row["sum_r"]) - n * self.bbox[0]
        sc = int(row["sum_c"]) - n * self.bbox[1]
        self._mu = (Fraction(n * int(row["m_rr"]) - sr * sr, n), Fraction(n * int(row["m_cc"]) - sc * sc, n),
                    Fraction(n * int(row["m_rc"]) - sr * sc, n))

    @property
    def inertia_tensor(self) -> np.ndarray:
        """skimage's inertia_tensor: [[mu_cc, -mu_rc], [-mu_rc, mu_rr]] / mu_00"""
        mu_rr, mu_cc, mu_rc = self._mu
        n = self.area
        return np.array([[float(mu_cc / n), float(-mu_rc / n)], [float(-mu_rc / n), float(mu_rr / n)]])

    @property
    def eccentricity(self) -> float:
        """skimage's eccentricity: sqrt(1 - l2 / l1) of the inertia tensor's eigenvalues (clipped at 0, decreasing), 0 if l1 is 0"""
        ev = np.clip(np.linalg.eigvalsh(self.inertia_tensor), 0, None)
        l1, l2 = sorted(ev, reverse=True)
        if l1 == 0:
            return 0
        return float(np.sqrt(1 - l2 / l1))


class Slice:
    """ct.py:321-441: one slice of a CatPhanBase series.  Its phantom outline is the series' localization row."""

    def __init__(self, catphan, slice_num: int | None = None, clear_borders: bool = True):
        if slice_num is not None:
            self.slice_num = slice_num
        self.image = catphan.dicom_stack[self.slice_num]
        self.mm_per_pixel = catphan.mm_per_pixel
        self.clear_borders = clear_borders
        self._catphan = catphan

    @property
    def phantom_row(self):
        """the slice's epid_ct_localize row (status, area, centroid)"""
        return self._catphan.localization(self.clear_borders)[self.slice_num]

    def is_phantom_in_view(self) -> bool:
        """Whether the phantom appears to be within the slice."""
        return int(self.phantom_row["status"]) == nat.CT_OK

    @property
    def phan_center(self) -> Point:
        """Determine the location of the center of the phantom."""
        fx, fy = self._catphan._phantom_center_func
        return Point(x=fx(self.slice_num), y=fy(self.slice_num))


class CatPhanBase:
    """ct.py:2027-2584: a CT phantom series and its localization (axis, origin slice).  The phantom classes add the roll and modules."""

    air_bubble_radius_mm: int | float = 7
    localization_radius: int | float = 59
    min_num_images = 39
    clear_borders: bool = True
    hu_origin_slice_variance = 400
    clip_in_localization: bool = False
    catphan_radius_mm: float
    x_adjustment: float = 0
    y_adjustment: float = 0
    angle_adjustment: float = 0
    roi_size_factor: float = 1
    scaling_factor: float = 1
    roll_slice_offset: float = 0

    def __init__(self, folderpath, check_uid: bool = True, memory_efficient_mode: bool = False, is_zip: bool = False):
        """folderpath: a folder, a list of files, or (is_zip) a zip archive of the series."""
        super().__init__()
        self.origin_slice = 0
        self.catphan_roll = 0
        self._phantom_center_func = None
        self._localization = {}
        if isinstance(folderpath, (str, Path)) and not is_zip:
            if not osp.isdir(folderpath):
                raise NotADirectoryError("Path given was not a Directory/Folder")
        if memory_efficient_mode:
            raise NotImplementedError("memory_efficient_mode (a lazily loaded series) is not supported; the series is read at once")
        if is_zip:
            self.dicom_stack = DicomImageStack.from_zip(folderpath, check_uid=check_uid, min_number=self.min_num_images)
        else:
            self.dicom_stack = DicomImageStack(folderpath, check_uid=check_uid, min_number=self.min_num_images)

    @classmethod
    def from_zip(cls, zip_file, check_uid: bool = True, memory_efficient_mode: bool = False):
        """Construct from a zip archive of the series."""
        return cls(folderpath=zip_file, check_uid=check_uid, memory_efficient_mode=memory_efficient_mode, is_zip=True)

    def _rescale(self) -> tuple[list[float], list[float]]:
        """Each slice's RescaleSlope and RescaleIntercept.  A series whose PixelIntensityRelationshipSign is -1 raises
        NotImplementedError."""
        slope, intercept = [], []
        for m in self.dicom_stack.metadatas:
            if m.get("PixelIntensityRelationshipSign") == -1:
                # the images are inverted after the rescale (core.image._rescale_dicom_values); the localization reads the
                # rescaled values only
                raise NotImplementedError("CT series with PixelIntensityRelationshipSign -1 (inverted pixel values) are not "
                                          "supported")
            s, i = m.get("RescaleSlope"), m.get("RescaleIntercept")
            # without both tags the image keeps its stored values, which (1, 0) reproduces exactly
            slope.append(1.0 if s is None or i is None else float(s))
            intercept.append(0.0 if s is None or i is None else float(i))
        return slope, intercept

    @property
    def _otsu_disk_radius(self) -> float:
        """get_regions' Otsu disk of a Slice, in pixels (ct.py:3334)"""
        return OTSU_DISK_RADIUS_MM / self.mm_per_pixel

    def localization(self, clear_borders: bool) -> np.ndarray:
        """The epid_ct_localize row of every slice (nat.CT_SLICE_DTYPE), computed once per clear_borders setting from the stored
        pixels and each slice's RescaleSlope / RescaleIntercept, on get_regions' ndarray branch (clip_in_localization) or its
        Slice branch."""
        if clear_borders not in self._localization:
            slope, intercept = self._rescale()
            self._localization[clear_borders] = nat.ct_localize(
                nat.Context.default(), self.dicom_stack.volume, slope, intercept, np.arange(self.num_images), self.catphan_size,
                clear_borders, self.clip_in_localization,
                otsu_disk_radius=0.0 if self.clip_in_localization else self._otsu_disk_radius)
        return self._localization[clear_borders]

    def get_regions(self, slice_num: int) -> list[Region]:
        """ct.py:3315-3348 get_regions(Slice(self, slice_num)) with its defaults: the regions in label order"""
        slope, intercept = self._rescale()
        rows, _, _ = nat.ct_regions(nat.Context.default(), self.dicom_stack.volume, slope, intercept, slice_num,
                                    self._otsu_disk_radius)
        return [Region(r) for r in rows]

    def localize(self, origin_slice: int | None) -> None:
        """Find the phantom axis, the origin slice and the roll, then check that the scan covers every module."""
        self._phantom_center_func = self.find_phantom_axis()
        if origin_slice is not None:
            self.origin_slice = origin_slice
        else:
            self.origin_slice = self.find_origin_slice()
        self.catphan_roll = self.find_phantom_roll() + self.angle_adjustment
        if origin_slice is None:
            self.origin_slice = self.refine_origin_slice(initial_slice_num=self.origin_slice)
        # now that we have the origin slice, ensure we have scanned all linked modules
        if not self._ensure_physical_scan_extent():
            raise ValueError(
                "The physical scan extent does not match the module configuration. "
                "This means not all modules were included in the scan. Rescan the phantom to include all"
                "relevant modules, or remove modules from the analysis."
            )

    def _module_offsets(self) -> list[float]:
        """The z of every module (the origin slice's z plus each module's offset); the phantom classes define it."""
        raise NotImplementedError

    def _ensure_physical_scan_extent(self) -> bool:
        """Whether the z of every module lies within the scanned z range, each rounded to 0.1 mm."""
        z_positions = [z_position(m) for m in self.dicom_stack.metadatas]
        min_scan_extent_slice = round(min(z_positions), 1)
        max_scan_extent_slice = round(max(z_positions), 1)
        min_config_extent_slice = round(min(self._module_offsets()), 1)
        max_config_extent_slice = round(max(self._module_offsets()), 1)
        return (min_config_extent_slice >= min_scan_extent_slice) and (max_config_extent_slice <= max_scan_extent_slice)

    def refine_origin_slice(self, initial_slice_num: int) -> int:
        """The identity here; phantoms may refine the origin slice."""
        return initial_slice_num

    def _is_right_area(self, region) -> bool:
        thresh = np.pi * ((self.air_bubble_radius_mm / self.mm_per_pixel) ** 2)
        return thresh * 2 > region.filled_area > thresh / 2

    def _is_right_eccentricity(self, region) -> bool:
        return region.eccentricity < 0.5

    def find_phantom_roll(self, func: Callable | None = None) -> float:
        """The roll in degrees from the two air bubbles of the slice roll_slice_offset mm from the origin slice: of the regions of the
        right area and eccentricity, the first two by `func` (default: closest to the phantom centre in x), top to bottom."""
        slice_offset = round(self.roll_slice_offset / self.dicom_stack.slice_spacing)
        slice_num = self.origin_slice + slice_offset
        slice = Slice(self, slice_num, clear_borders=self.clear_borders)
        regions = self.get_regions(slice_num)
        hu_bubbles = [r for r in regions if (self._is_right_area(r) and self._is_right_eccentricity(r))]
        func = func or (lambda x: abs(x.centroid[1] - slice.phan_center.x))
        central_bubbles = sorted(hu_bubbles, key=func)[:2]
        sorted_bubbles = sorted(central_bubbles, key=lambda x: x.centroid[0])  # top, bottom
        if len(sorted_bubbles) < 2:
            warnings.warn("Could not determine phantom roll. Setting roll to 0.", UserWarning)
            return 0.0
        y_dist = sorted_bubbles[1].centroid[0] - sorted_bubbles[0].centroid[0]
        x_dist = sorted_bubbles[1].centroid[1] - sorted_bubbles[0].centroid[1]
        phan_roll = np.arctan2(y_dist, x_dist)
        anglroll = np.rad2deg(phan_roll) - 90
        return anglroll

    def find_phantom_axis(self):
        """Fit the phantom centres of every slice where the phantom is in view to two lines in z (np.polyfit, deg 1)."""
        rows = self.localization(self.clear_borders)
        z, center_x, center_y = [], [], []
        for idx, row in enumerate(rows):
            if int(row["status"]) == nat.CT_OK:
                z.append(idx)
                center_y.append(row["centroid_row"])
                center_x.append(row["centroid_col"])
        zs = np.array(z)
        center_xs = np.array(center_x) + self.x_adjustment
        center_ys = np.array(center_y) + self.y_adjustment
        x_idxs = np.argwhere(np.isclose(np.median(center_xs), center_xs, atol=3, rtol=0.01))
        y_idxs = np.argwhere(np.isclose(np.median(center_ys), center_ys, atol=3, rtol=0.01))
        common_idxs = np.intersect1d(x_idxs, y_idxs)
        fit_zx = np.poly1d(np.polyfit(zs[common_idxs], center_xs[common_idxs], deg=1, rcond=0.00001))
        fit_zy = np.poly1d(np.polyfit(zs[common_idxs], center_ys[common_idxs], deg=1, rcond=0.00001))
        return fit_zx, fit_zy

    @property
    def mm_per_pixel(self) -> float:
        """The millimeters per pixel of the DICOM images."""
        return self.dicom_stack.metadata.PixelSpacing[0]

    def _hu_profile(self, image_number: int):
        """the collapsed circle profile find_origin_slice reads on slice image_number, or None when the phantom is not in view"""
        slice = Slice(self, image_number, clear_borders=self.clear_borders)
        if not slice.is_phantom_in_view():
            return None
        return CollapsedCircleProfile(slice.phan_center, radius=self.localization_radius / self.mm_per_pixel,
                                      image_array=slice.image.array, width_ratio=0.05, num_profiles=5).values

    def find_origin_slice(self) -> int:
        """The median of the even slices whose circle profile looks like the HU module."""
        hu_slices = []
        for image_number in range(0, self.num_images, 2):
            prof = self._hu_profile(image_number)
            if prof is not None:
                low_end, high_end = np.percentile(prof, [2, 98])
                median = np.median(prof)
                middle_variation = np.percentile(prof, 80) - np.percentile(prof, 20)
                variation_limit = max(100, self.dicom_stack.metadata.SliceThickness * -100 + 300)
                if ((low_end < median - self.hu_origin_slice_variance) and (high_end > median + self.hu_origin_slice_variance)
                        and (middle_variation < variation_limit)):
                    hu_slices.append(image_number)
        return self._center_hu_slice(hu_slices)

    def _center_hu_slice(self, hu_slices: list) -> int:
        if not hu_slices:
            raise ValueError("No slices were found that resembled the HU linearity module")
        hu_slices = np.array(hu_slices)
        c = int(round(float(np.median(hu_slices))))
        ln = len(hu_slices)
        hu_slices = hu_slices[((c + ln / 2) >= hu_slices) & (hu_slices >= (c - ln / 2))]
        center_hu_slice = int(round(float(np.median(hu_slices))))
        if self._is_within_image_extent(center_hu_slice):
            return center_hu_slice

    @property
    def num_images(self) -> int:
        """The number of images loaded."""
        return len(self.dicom_stack)

    def _is_within_image_extent(self, image_num: int) -> bool:
        """Determine if the image number is beyond the edges of the images (negative or past last image)."""
        if self.num_images - 1 > image_num > 1:
            return True
        raise ValueError("The determined image number is beyond the image extent. Either the entire dataset "
                         "wasn't loaded or the entire phantom wasn't scanned.")

    @property
    def catphan_size(self) -> float:
        """The expected size of the phantom in pixels."""
        phan_area = np.pi * (self.catphan_radius_mm**2)
        return phan_area / (self.mm_per_pixel**2)


class ROIResult(BaseModel):
    """ct.py:85-99: one ROI of a module in results_data()."""

    name: str
    value: float
    stdev: float
    difference: float | None
    nominal_value: float | None
    passed: bool | None


class HUDiskROI(DiskROI):
    """ct.py:251-297: a disk ROI of an HU sample or uniformity region, with its nominal value and tolerance."""

    def __init__(self, array, angle: float, roi_radius: float, dist_from_center: float, phantom_center: tuple | Point,
                 nominal_value: float | None = None, tolerance: float | None = None, background_mean: float | None = None,
                 background_std: float | None = None):
        new_center = self._get_shifted_center(angle, dist_from_center, phantom_center)
        super().__init__(array, roi_radius, new_center)
        self.nominal_val = nominal_value
        self.tolerance = tolerance

    @property
    def value_diff(self) -> float:
        """The difference in HU between measured and nominal."""
        return self.pixel_value - self.nominal_val

    @property
    def passed(self) -> bool:
        """Whether the ROI's pixel value is within tolerance of the nominal value."""
        if self.tolerance:
            return abs(self.value_diff) <= self.tolerance
        return True

    @property
    def plot_color(self) -> str:
        return "green" if self.passed else "red"


class CatPhanModule(Slice):
    """ct.py:443-623: a module of the phantom on one slice, `offset` mm from the origin slice, with its disk ROIs.  The ROIs'
    statistics come from one ``fill_disk_stats`` call.  Like the reference, ``_convert_units_in_settings`` writes the pixel values
    into the class's own ``roi_settings`` dicts, so they show in ``results_data()`` and the last instance's values stay there."""

    common_name: str = ""
    combine_method: str = "mean"
    num_slices: int = 0
    roi_settings: dict = {}
    background_roi_settings: dict = {}
    roi_dist_mm = float
    roi_radius_mm = float
    rois: dict = {}
    background_rois: dict = {}
    window_min: int | None = None
    window_max: int | None = None

    def __init__(self, catphan, tolerance: float | None = None, offset: int = 0, clear_borders: bool = True):
        self.model = ""
        self._offset = offset
        self.origin_slice = catphan.origin_slice
        self.tolerance = tolerance
        self.slice_thickness = catphan.dicom_stack.metadata.SliceThickness
        self.slice_spacing = catphan.dicom_stack.slice_spacing
        self.catphan_roll = catphan.catphan_roll
        self.roi_size_factor = catphan.roi_size_factor
        self.scaling_factor = catphan.scaling_factor
        self.roll_slice_offset = catphan.roll_slice_offset
        self.rois: dict[str, HUDiskROI] = {}
        self.background_rois: dict[str, HUDiskROI] = {}
        if self.num_slices > 0:
            raise NotImplementedError("modules that combine the surrounding slices (num_slices > 0) are not supported")
        Slice.__init__(self, catphan, clear_borders=clear_borders)
        self._convert_units_in_settings()
        self.preprocess(catphan)
        self._setup_rois()
        fill_disk_stats([*self.background_rois.values(), *self.rois.values()])

    def _convert_units_in_settings(self) -> None:
        setting_groups = [getattr(self, attr) for attr in dir(self) if attr.endswith("roi_settings")]
        for roi_settings in setting_groups:
            for roi, settings in roi_settings.items():
                if isinstance(settings, dict):
                    if settings.get("distance") is not None:
                        settings["distance_pixels"] = settings["distance"] * self.scaling_factor / self.mm_per_pixel
                    if settings.get("radial_distance") is not None:
                        settings["radial_distance_pixels"] = settings["radial_distance"] * self.scaling_factor / self.mm_per_pixel
                    if settings.get("transversal_distance") is not None:
                        settings["transversal_distance_pixels"] = (settings["transversal_distance"] * self.scaling_factor
                                                                   / self.mm_per_pixel)
                    if settings.get("angle") is not None:
                        settings["angle_corrected"] = settings["angle"] + self.catphan_roll
                    if settings.get("radius") is not None:
                        settings["radius_pixels"] = settings["radius"] * self.roi_size_factor / self.mm_per_pixel
                    if settings.get("width") is not None:
                        settings["width_pixels"] = settings["width"] * self.roi_size_factor / self.mm_per_pixel
                    if settings.get("height") is not None:
                        settings["height_pixels"] = settings["height"] * self.roi_size_factor / self.mm_per_pixel

    def preprocess(self, catphan):
        """A preprocessing step before the ROIs are placed."""

    @property
    def slice_num(self) -> int:
        """The module's slice: the origin slice plus the offset in slices."""
        return int(self.origin_slice + round(self._offset / self.slice_spacing))

    def _setup_rois(self) -> None:
        for name, setting in self.background_roi_settings.items():
            self.background_rois[name] = HUDiskROI(self.image, setting["angle_corrected"], setting["radius_pixels"],
                                                   setting["distance_pixels"], self.phan_center)
        for name, setting in self.roi_settings.items():
            nominal_value = setting.get("value", 0)
            # the reference passes the background ROIs' mean and std here, which HUDiskROI does not keep
            self.rois[name] = HUDiskROI(self.image, setting["angle_corrected"], setting["radius_pixels"], setting["distance_pixels"],
                                        self.phan_center, nominal_value, self.tolerance)

    @property
    def roi_vals_as_str(self) -> str:
        return ", ".join(f"{name}: {roi.pixel_value}" for name, roi in self.rois.items())


def rois_to_results(dict_mapping: dict[str, DiskROI]) -> dict[str, ROIResult]:
    """ct.py:3389-3401: ROIs -> ROIResults, for results_data."""
    flat_dict = {}
    for name, roi in dict_mapping.items():
        flat_dict[name] = ROIResult(name=name, value=roi.pixel_value, stdev=roi.std, difference=getattr(roi, "value_diff", None),
                                    nominal_value=getattr(roi, "nominal_val", None), passed=getattr(roi, "passed", None))
    return flat_dict
