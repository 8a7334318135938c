"""pylinac.cheese (cheese.py:23-775): the TomoTherapy "cheese" phantom and the CIRS 062M electron-density phantom.

The localization is pylinac_b200.ct's (one device pass over the series); the roll is a collapsed circle profile on the device with the
reference's peak search; the module's disk ROIs are computed in one ``fill_disk_stats`` call on the float64 HU origin slice.  Plots,
PDF reports and demo images are not provided.
"""
from __future__ import annotations

from collections.abc import Callable

import numpy as np
from pydantic import Field

from .core.profile import CollapsedCircleProfile
from .core.roi import DiskROI, fill_disk_stats
from .core.utilities import ResultBase, ResultsDataMixin
from .core.warnings import capture_warnings
from .ct import CatPhanBase, Slice


def wrap360(value):
    """core/scale.py:23-25"""
    return value % 360


class TomoCheeseResult(ResultBase):
    """Returned by ``TomoCheese.results_data()``."""

    origin_slice: int = Field(description="The slice index that was used for the ROI analysis.", title="Slice number of the analyzed image")
    num_images: int = Field(description="The number of images that were in the passed dataset.", title="Number of images in the stack")
    phantom_roll: float = Field(description="The roll of the phantom in degrees.", title="Phantom roll (\N{DEGREE SIGN})")
    rois: dict[str, dict[str, int | float]] = Field(description="A dictionary of measured ROIs.", title="ROI data")
    roi_1: dict = Field(title="ROI 1")
    roi_2: dict = Field(title="ROI 2")
    roi_3: dict = Field(title="ROI 3")
    roi_4: dict = Field(title="ROI 4")
    roi_5: dict = Field(title="ROI 5")
    roi_6: dict = Field(title="ROI 6")
    roi_7: dict = Field(title="ROI 7")
    roi_8: dict = Field(title="ROI 8")
    roi_9: dict = Field(title="ROI 9")
    roi_10: dict = Field(title="ROI 10")
    roi_11: dict = Field(title="ROI 11")
    roi_12: dict = Field(title="ROI 12")
    roi_13: dict = Field(title="ROI 13")
    roi_14: dict = Field(title="ROI 14")
    roi_15: dict = Field(title="ROI 15")
    roi_16: dict = Field(title="ROI 16")
    roi_17: dict = Field(title="ROI 17")
    roi_18: dict = Field(title="ROI 18")
    roi_19: dict = Field(title="ROI 19")
    roi_20: dict = Field(title="ROI 20")


class CheeseResult(ResultBase):
    """Returned by ``CIRS062M.results_data()``."""

    origin_slice: int = Field(description="The slice index that was used for the ROI analysis.", title="Slice number of the analyzed image")
    num_images: int = Field(description="The number of images that were in the passed dataset.", title="Number of images in the stack")
    phantom_roll: float = Field(description="The roll of the phantom in degrees.", title="Phantom roll (\N{DEGREE SIGN})")
    rois: dict[str, dict[str, int | float]] = Field(description="A dictionary of measured ROIs.", title="ROI data")


class CheeseModule(Slice):
    """cheese.py:91-122 with ct.py:443-534: the one module of a cheese-like phantom, on the origin slice, with a disk ROI per insert."""

    common_name: str
    roi_settings: dict[str, dict[str, float]]

    def __init__(self, catphan, clear_borders: bool = True):
        self.origin_slice = catphan.origin_slice
        self.catphan_roll = catphan.catphan_roll
        self.roi_size_factor = catphan.roi_size_factor
        self.scaling_factor = catphan.scaling_factor
        self.mm_per_pixel = catphan.mm_per_pixel
        super().__init__(catphan, self.origin_slice, clear_borders=clear_borders)
        self.rois: dict[str, DiskROI] = {}
        for name, s in self.roi_settings.items():
            self.rois[name] = DiskROI.from_phantom_center(
                self.image, s["angle"] + self.catphan_roll, s["radius"] * self.roi_size_factor / self.mm_per_pixel,
                s["distance"] * self.scaling_factor / self.mm_per_pixel, self.phan_center)
        fill_disk_stats(list(self.rois.values()))


class TomoCheeseModule(CheeseModule):
    """The pluggable module with user-accessible holes: the inner circle (65 mm) ~45 degrees apart, the outer (110 mm) ~30 degrees
    apart, radius 12 mm."""

    common_name = "Tomo Cheese"
    inner_roi_dist_mm = 65
    outer_roi_dist_mm = 110
    roi_radius_mm = 12
    roi_settings = {
        name: {"angle": angle, "distance": 110 if outer else 65, "radius": 12}
        for name, angle, outer in [
            ("1", -75, True), ("2", -67.5, False), ("3", -45, True), ("4", -22.5, False), ("5", -15, True), ("6", 15, True),
            ("7", 22.5, False), ("8", 45, True), ("9", 67.5, False), ("10", 75, True), ("11", 105, True), ("12", 112.5, False),
            ("13", 135, True), ("14", 157.5, False), ("15", 165, True), ("16", -165, True), ("17", -157.5, False), ("18", -135, True),
            ("19", -112.5, False), ("20", -105, True)]
    }


class CIRSHUModule(CheeseModule):
    """The pluggable module with user-accessible holes, each circle (60 mm, 115 mm) ~45 degrees apart, radius 10 mm."""

    common_name = "CIRS electron density"
    outer_radius_mm = 115
    inner_radius_mm = 60
    roi_radius_mm = 10
    roi_settings = {
        name: {"angle": angle, "distance": distance, "radius": 10}
        for name, angle, distance in [
            ("1", 0, 0), ("2", -90, 60), ("3", -90, 115), ("4", -45, 60), ("5", -45, 115), ("6", 0, 60), ("7", 0, 115), ("8", 45, 60),
            ("9", 45, 115), ("10", 90, 60),
            # closer to the ring; presumably because the bottom of the phantom is flatter than the top
            ("11", 90, 110),
            ("12", 135, 60), ("13", 135, 115), ("14", 180, 60), ("15", 180, 115), ("16", -135, 60), ("17", -135, 115)]
    }


class CheesePhantomBase(CatPhanBase, ResultsDataMixin[CheeseResult]):
    """cheese.py:240-552: a cheese-like phantom, one module."""

    model: str
    air_bubble_radius_mm: int | float
    localization_radius: int | float
    min_num_images: int
    catphan_radius_mm: float
    roi_config: dict
    module_class: type[CheeseModule]
    module: CheeseModule
    clip_in_localization = True

    def analyze(self, roi_config: dict | None = None, x_adjustment: float = 0, y_adjustment: float = 0, angle_adjustment: float = 0,
                roi_size_factor: float = 1, scaling_factor: float = 1, origin_slice: int | None = None) -> None:
        """Analyze the phantom.  x / y_adjustment move the detected centre (pixels), angle_adjustment adds to the roll (degrees),
        roi_size_factor scales the ROI radii and scaling_factor their distances from the centre; origin_slice overrides the detected
        HU slice."""
        self.x_adjustment = x_adjustment
        self.y_adjustment = y_adjustment
        self.angle_adjustment = angle_adjustment
        self.roi_size_factor = roi_size_factor
        self.scaling_factor = scaling_factor
        self.localize(origin_slice=origin_slice)
        self.module = self.module_class(self, clear_borders=self.clear_borders)
        self.roi_config = roi_config

    def _ensure_physical_scan_extent(self) -> bool:
        """cheese.py:303-305: a cheese phantom has one module, always in the scan."""
        return True

    def _roi_angles(self) -> list[float]:
        return [wrap360(s["angle"]) for s in self.module_class.roi_settings.values()]

    def find_phantom_roll(self, func: Callable | None = None) -> float:
        """The shift of the highest insert on the outer circle to the nearest nominal insert angle, if within 5 degrees; else 0."""
        slice = Slice(self, self.origin_slice, clear_borders=self.clear_borders)
        circle = CollapsedCircleProfile(slice.phan_center, self.localization_radius / self.mm_per_pixel, slice.image.array, ccw=False,
                                        width_ratio=0.05, num_profiles=5)
        # we only want peaks. air pockets can cause bad range shifts so set min to 0
        circle.values = np.where(circle.values < 0, 0, circle.values)
        peak_idxs, _ = circle.find_fwxm_peaks(max_number=1)
        if peak_idxs:
            angle = peak_idxs[0] / len(circle.values) * 360
            shifts = [angle - a for a in self._roi_angles()]
            min_shift = shifts[np.argmin([abs(shift) for shift in shifts])]
            if -5 < min_shift < 5:
                return min_shift
            print(f"Detected shift of {min_shift} was >5 degrees; automatic roll compensation aborted. Setting roll to 0.")
            return 0
        print("No low-HU regions found in the outer ROI circle; automatic roll compensation aborted. Setting roll to 0.")
        return 0

    def results(self, as_list: bool = False) -> str | list[str]:
        """The results of the analysis as a string (or a list of lines)."""
        results = [f" - {self.model} Phantom Analysis - ", " - HU Module - "]
        results += [f"ROI {name} median: {roi.pixel_value:.1f}, stdev: {roi.std:.1f}" for name, roi in self.module.rois.items()]
        if as_list:
            return results
        return "\n".join(results)

    def _generate_results_data(self) -> CheeseResult:
        return CheeseResult(origin_slice=self.origin_slice, num_images=self.num_images, phantom_roll=self.catphan_roll,
                            rois={name: roi.as_dict() for name, roi in self.module.rois.items()})


@capture_warnings
class TomoCheese(CheesePhantomBase, ResultsDataMixin[TomoCheeseResult]):
    """The TomoTherapy 'Cheese' phantom: insert holes and plugs for HU analysis."""

    model = "Tomotherapy Cheese"
    air_bubble_radius_mm = 14
    localization_radius = 110
    min_num_images = 10
    catphan_radius_mm = 150
    module_class = TomoCheeseModule
    module: TomoCheeseModule

    def _generate_results_data(self):
        rois = {name: roi.as_dict() for name, roi in self.module.rois.items()}
        return TomoCheeseResult(origin_slice=self.origin_slice, num_images=self.num_images, phantom_roll=self.catphan_roll, rois=rois,
                                **{f"roi_{k}": self.module.rois[str(k)].as_dict() for k in range(1, 21)})


@capture_warnings
class CIRS062M(CheesePhantomBase):
    """The CIRS electron density phantom (062M): insert holes and plugs for HU analysis."""

    model = "CIRS Electron Density (062M)"
    air_bubble_radius_mm = 30
    clear_borders = False
    hu_origin_slice_variance = 150
    localization_radius = 115
    catphan_radius_mm = 155
    min_num_images = 10
    module_class = CIRSHUModule
    module: CIRSHUModule

    def find_origin_slice(self) -> int:
        """The reference's override: a lower variation limit, and its condition as Python groups it, a or (b and c)."""
        hu_slices = []
        for image_number in range(0, self.num_images, 2):
            prof = self._hu_profile(image_number)
            if prof is not None:
                low_end, high_end = np.percentile(prof, [2, 98])
                median = np.median(prof)
                middle_variation = np.percentile(prof, 60) - np.percentile(prof, 40)
                variation_limit = max(100, self.dicom_stack.metadata.SliceThickness * -100 + 300)
                if ((low_end < median - self.hu_origin_slice_variance)
                        or (high_end > median + self.hu_origin_slice_variance) and (middle_variation < variation_limit)):
                    hu_slices.append(image_number)
        return self._center_hu_slice(hu_slices)
