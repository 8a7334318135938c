"""pylinac.ct's CatPhanBase localization (ct.py:321-441, 2027-2584), as far as the cheese phantoms use it.

One ``epid_ct_localize`` call (csrc/ct.cu) finds the phantom outline in every slice of the series: Slice.phantom_roi's Scharr edges,
Gaussian smoothing, Otsu threshold, clear_border, binary_fill_holes, labelling and region choice, bit-identical to the reference.
``find_phantom_axis`` (every slice) and ``find_origin_slice`` (every other slice) both read its rows, where the reference runs the
per-slice pipeline twice.  The axis fit, the circle-profile percentiles and the origin choice are the reference's own numpy calls on
the host; the circle profiles run on the device (core.profile).
"""
from __future__ import annotations

import os.path as osp
from pathlib import Path

import numpy as np

from . import _native as nat
from .core.geometry import Point
from .core.image import DicomImageStack
from .core.profile import CollapsedCircleProfile


class Slice:
    """ct.py:321-441: one slice of a CatPhanBase series.  Its phantom outline is the series' localization row."""

    def __init__(self, catphan, slice_num: int, clear_borders: bool = True):
        self.slice_num = slice_num
        self.image = catphan.dicom_stack[slice_num]
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

    def localization(self, clear_borders: bool) -> np.ndarray:
        """The epid_ct_localize row of every slice (nat.CT_SLICE_DTYPE), computed once per clear_borders setting from the stored
        pixels and each slice's RescaleSlope / RescaleIntercept.  A series whose PixelIntensityRelationshipSign is -1 raises
        NotImplementedError."""
        if clear_borders not in self._localization:
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
            self._localization[clear_borders] = nat.ct_localize(
                nat.Context.default(), self.dicom_stack.volume, slope, intercept, np.arange(self.num_images), self.catphan_size,
                clear_borders, self.clip_in_localization)
        return self._localization[clear_borders]

    def localize(self, origin_slice: int | None) -> None:
        """Find the phantom axis, the origin slice and the roll.  (The reference's refine_origin_slice and scan-extent check are the
        identity and True for the cheese phantoms.)"""
        self._phantom_center_func = self.find_phantom_axis()
        if origin_slice is not None:
            self.origin_slice = origin_slice
        else:
            self.origin_slice = self.find_origin_slice()
        self.catphan_roll = self.find_phantom_roll() + self.angle_adjustment

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
