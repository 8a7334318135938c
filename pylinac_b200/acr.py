"""pylinac.acr's ACR CT 464 phantom (acr.py:39-698): four modules, each a set of disk ROIs on one slice.

The phantom is located by pylinac_b200.ct on get_regions' Slice branch (one device pass over the series), its roll from the two air
bubbles of the HU module (one ``epid_ct_regions`` call), and each module's ROI statistics in one ``fill_disk_stats`` call on the
float64 HU slice.  The MTF is core.mtf.MTF on the resolution disks' maxima and minima.  Plots, PDF reports and QuAAC output are not
provided, nor is the ACR MRI phantom.
"""
from __future__ import annotations

from pydantic import BaseModel, Field

from .core.mtf import MTF
from .core.roi import HighContrastDiskROI
from .core.utilities import ResultBase, ResultsDataMixin
from .core.warnings import capture_warnings
from .ct import CatPhanBase, CatPhanModule, z_position

CT_UNIFORMITY_MODULE_OFFSET_MM = 70
CT_SPATIAL_RESOLUTION_MODULE_OFFSET_MM = 100
CT_LOW_CONTRAST_MODULE_OFFSET_MM = 30


class CTModule(CatPhanModule):
    """The HU linearity module: five material inserts."""

    common_name = "HU Linearity"
    attr_name = "ct_calibration_module"
    roi_dist_mm = 63
    roi_radius_mm = 10
    roi_settings = {
        "Air": {"angle": 45, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Poly": {"angle": 225, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Acrylic": {"angle": 135, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Bone": {"angle": -45, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Water": {"angle": 180, "distance": roi_dist_mm, "radius": roi_radius_mm},
    }
    window_min = -200
    window_max = 200


class CTModuleOutput(BaseModel):
    """A module of ``ACRCT.results_data()``."""

    offset: float = Field(description="The offset of the module slice in mm from the origin slice (z-direction).")
    roi_distance_from_center_mm: float = Field(
        description="The distance of the ROIs from the center of the phantom in mm in the image plane.")
    roi_radius_mm: float = Field(description="The radius of the ROIs in mm.")
    roi_settings: dict = Field(description="The ROI settings. The keys are the material names.")
    rois: dict[str, float] = Field(
        description="The analyzed ROIs. The key is the name of the material and the value is the mean HU value. E.g. ``'Air': -987.1``.")


class UniformityModule(CatPhanModule):
    """The uniformity module: five ROIs that should all read the same value."""

    attr_name = "uniformity_module"
    common_name = "HU Uniformity"
    roi_dist_mm = 66
    roi_radius_mm = 11
    roi_settings = {
        "Top": {"angle": -90, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Right": {"angle": 0, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Bottom": {"angle": 90, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Left": {"angle": 180, "distance": roi_dist_mm, "radius": roi_radius_mm},
        "Center": {"angle": 0, "distance": 0, "radius": roi_radius_mm},
    }
    window_min = -50
    window_max = 50


class UniformityModuleOutput(CTModuleOutput):
    """The uniformity module of ``ACRCT.results_data()``."""

    center_roi_stdev: float = Field(description="The standard deviation of the center ROI.", title="Center ROI Standard Deviation")


class SpatialResolutionModule(CatPhanModule):
    """The spatial resolution module: eight high-contrast bar patterns, 0.4 to 1.2 lp/mm."""

    attr_name = "spatial_resolution_module"
    common_name = "Spatial Resolution"
    rois: dict[str, HighContrastDiskROI]
    roi_dist_mm = 70
    roi_radius_mm = 6
    roi_settings = {
        "10oclock": {"angle": -135, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 0.4},
        "9oclock": {"angle": -180, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 0.5},
        "7oclock": {"angle": 135, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 0.6},
        "6oclock": {"angle": 90, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 0.7},
        "4oclock": {"angle": 45, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 0.8},
        "3oclock": {"angle": 0, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 0.9},
        "2oclock": {"angle": -45, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 1.0},
        "12oclock": {"angle": -90, "distance": roi_dist_mm, "radius": roi_radius_mm, "lp/mm": 1.2},
    }

    def _setup_rois(self) -> None:
        for name, setting in self.roi_settings.items():
            self.rois[name] = HighContrastDiskROI.from_phantom_center(
                self.image, setting["angle_corrected"], setting["radius_pixels"], setting["distance_pixels"], self.phan_center,
                contrast_threshold=1.0)  # fixed to 1 so everything passes; no pass/fail here

    @property
    def mtf(self) -> MTF:
        spacings = [roi["lp/mm"] for roi in self.roi_settings.values()]
        return MTF.from_high_contrast_diskset(spacings=spacings, diskset=list(self.rois.values()))


class SpatialResolutionModuleOutput(CTModuleOutput):
    """The spatial resolution module of ``ACRCT.results_data()``."""

    lpmm_to_rmtf: dict = Field(
        description="Line pair to relative modulation transfer mapping. The keys are the line pair values and the values are the "
                    "relative modulation transfer values.", title="Line Pair to Relative MTF")


class LowContrastModule(CatPhanModule):
    """The low-contrast module: one contrast ROI and one background ROI."""

    attr_name = "low_contrast_module"
    common_name = "Low Contrast"
    roi_dist_mm = 60
    roi_radius_mm = 6
    nominal_value = 0
    roi_settings = {
        "ROI": {"angle": -90, "distance": roi_dist_mm, "radius": roi_radius_mm},
    }
    background_roi_settings = {
        "ROI": {"angle": -115, "distance": roi_dist_mm, "radius": roi_radius_mm},
    }
    window_min = 50
    window_max = 150

    def cnr(self) -> float:
        """|A - B| / SD, A the contrast ROI's median, B the background's and SD the background's standard deviation"""
        return abs(self.rois["ROI"].pixel_value - self.background_rois["ROI"].pixel_value) / self.background_rois["ROI"].std


class LowContrastModuleOutput(CTModuleOutput):
    """The low-contrast module of ``ACRCT.results_data()``."""

    cnr: float = Field(description="The contrast-to-noise ratio.", title="Contrast to Noise Ratio")


class ACRCTResult(ResultBase):
    """Returned by ``ACRCT.results_data()``."""

    phantom_model: str = Field(description="The model of the phantom used.")
    phantom_roll_deg: float = Field(description="The roll of the phantom in degrees.", title="Phantom roll (\N{DEGREE SIGN})")
    origin_slice: int = Field(description="The slice number of the 'origin' slice; for ACR this is Module 1.")
    num_images: int = Field(description="The number of images in the passed dataset.")
    ct_module: CTModuleOutput = Field(description="The results of the CT module.", title="CT Module")
    uniformity_module: UniformityModuleOutput = Field(description="The results of the Uniformity module.", title="HU Uniformity")
    low_contrast_module: LowContrastModuleOutput = Field(description="The results of the Low Contrast module.",
                                                         title="Low Contrast Resolution")
    spatial_resolution_module: SpatialResolutionModuleOutput = Field(description="The results of the Spatial Resolution module.",
                                                                     title="Spatial Resolution")


@capture_warnings
class ACRCT(CatPhanBase, ResultsDataMixin[ACRCTResult]):
    """The ACR CT 464 phantom: HU linearity, uniformity, spatial resolution and low contrast, each on one slice."""

    _model = "ACR CT 464"
    catphan_radius_mm = 100
    air_bubble_radius_mm = 14
    min_num_images = 4
    localization_radius = 70
    ct_calibration_module = CTModule
    low_contrast_module = LowContrastModule
    spatial_resolution_module = SpatialResolutionModule
    uniformity_module = UniformityModule
    clear_borders = False

    def _detected_modules(self) -> list[CatPhanModule]:
        return [self.ct_calibration_module, self.low_contrast_module, self.spatial_resolution_module, self.uniformity_module]

    def analyze(self, x_adjustment: float = 0, y_adjustment: float = 0, angle_adjustment: float = 0, roi_size_factor: float = 1,
                scaling_factor: float = 1, origin_slice: int | None = None) -> None:
        """Analyze the phantom.  x / y_adjustment move the detected centre (pixels), angle_adjustment adds to the roll (degrees),
        roi_size_factor scales the ROI radii and scaling_factor their distances from the centre; origin_slice overrides the detected
        HU linearity slice."""
        self.x_adjustment = x_adjustment
        self.y_adjustment = y_adjustment
        self.angle_adjustment = angle_adjustment
        self.roi_size_factor = roi_size_factor
        self.scaling_factor = scaling_factor
        self.localize(origin_slice=origin_slice)
        # each module class attribute is replaced by its instance, as in the reference: a second analyze() on the same object calls
        # the instance and raises TypeError
        self.ct_calibration_module = self.ct_calibration_module(self, offset=0, clear_borders=self.clear_borders)
        self.uniformity_module = self.uniformity_module(self, offset=CT_UNIFORMITY_MODULE_OFFSET_MM, clear_borders=self.clear_borders)
        self.spatial_resolution_module = self.spatial_resolution_module(self, offset=CT_SPATIAL_RESOLUTION_MODULE_OFFSET_MM,
                                                                        clear_borders=self.clear_borders)
        self.low_contrast_module = self.low_contrast_module(self, offset=CT_LOW_CONTRAST_MODULE_OFFSET_MM,
                                                            clear_borders=self.clear_borders)

    def find_phantom_roll(self, func=lambda roi: roi.bbox_area) -> float:
        """The roll from the two air bubbles, sorted by bbox area rather than by distance from the centre: both are right of it."""
        return super().find_phantom_roll(func)

    def results(self) -> str:
        """The results of the analysis as a string."""
        string = (
            f"\n - ACR CT 464 QA Test - \n"
            f"HU ROIs: {self.ct_calibration_module.roi_vals_as_str}\n"
            f"Contrast to Noise Ratio: {self.low_contrast_module.cnr():2.2f}\n"
            f"Uniformity ROIs: {self.uniformity_module.roi_vals_as_str}\n"
            f"Uniformity Center ROI standard deviation: {self.uniformity_module.rois['Center'].std:2.2f}\n"
            f"MTF 50% (lp/mm): {self.spatial_resolution_module.mtf.relative_resolution(50):2.2f}\n"
        )
        return string

    def _generate_results_data(self) -> ACRCTResult:
        ct, un, sr, lc = self.ct_calibration_module, self.uniformity_module, self.spatial_resolution_module, self.low_contrast_module
        return ACRCTResult(
            phantom_model="ACR CT 464",
            phantom_roll_deg=self.catphan_roll,
            origin_slice=self.origin_slice,
            num_images=self.num_images,
            ct_module=CTModuleOutput(offset=0, roi_distance_from_center_mm=ct.roi_dist_mm, roi_radius_mm=ct.roi_radius_mm,
                                     roi_settings=ct.roi_settings, rois={name: roi.mean for name, roi in ct.rois.items()}),
            uniformity_module=UniformityModuleOutput(
                offset=CT_UNIFORMITY_MODULE_OFFSET_MM, roi_distance_from_center_mm=un.roi_dist_mm, roi_radius_mm=un.roi_radius_mm,
                roi_settings=un.roi_settings, rois={name: roi.mean for name, roi in un.rois.items()},
                center_roi_stdev=un.rois["Center"].std),
            spatial_resolution_module=SpatialResolutionModuleOutput(
                offset=CT_SPATIAL_RESOLUTION_MODULE_OFFSET_MM, roi_distance_from_center_mm=sr.roi_dist_mm,
                roi_radius_mm=sr.roi_radius_mm, roi_settings=sr.roi_settings,
                rois={name: roi.pixel_value for name, roi in sr.rois.items()}, lpmm_to_rmtf=sr.mtf.norm_mtfs),
            low_contrast_module=LowContrastModuleOutput(
                offset=CT_LOW_CONTRAST_MODULE_OFFSET_MM, roi_distance_from_center_mm=lc.roi_dist_mm, roi_radius_mm=lc.roi_radius_mm,
                roi_settings=lc.roi_settings, rois={name: roi.pixel_value for name, roi in lc.rois.items()}, cnr=lc.cnr()),
        )

    def _module_offsets(self) -> list[float]:
        absolute_origin_position = z_position(self.dicom_stack.metadatas[self.origin_slice])
        relative_offsets_mm = [0, CT_UNIFORMITY_MODULE_OFFSET_MM, CT_LOW_CONTRAST_MODULE_OFFSET_MM, CT_SPATIAL_RESOLUTION_MODULE_OFFSET_MM]
        return [absolute_origin_position + offset_mm for offset_mm in relative_offsets_mm]

