"""Image classes mirroring ``pylinac.core.image`` (reference file cited per method) whose pixel arithmetic runs
in hand-written CUDA through ``libepid.so``.  Pure re-indexing (crop / flip / roll / rot90) stays a numpy view
operation exactly like the reference; everything that touches pixel values is a native call.
"""
from __future__ import annotations

import io
import os
import os.path as osp
from pathlib import Path
from typing import Any

import numpy as np

from .. import _native as nat
from .. import dicom
from . import array_utils as au
from .geometry import Point

MM_PER_INCH = 25.4


def _is_array(obj: Any) -> bool:
    return isinstance(obj, np.ndarray)


def _is_dicom(path) -> bool:
    try:
        return dicom.is_dicom(path)
    except Exception:
        return False


def _uniquify(seq, value: str) -> str:
    """core/utilities.py:368-377: value, value-1, value-2, ... until it is not in seq."""
    if value not in seq:
        return value
    i = 1
    while f"{value}-{i}" in seq:
        i += 1
    return f"{value}-{i}"


def _is_image_file(path) -> bool:
    """core/image.py:429-435: readable by Pillow."""
    try:
        from PIL import Image as pImage

        with pImage.open(path):
            return True
    except Exception:
        return False


def retrieve_image_files(path) -> list:
    """core/image.py:233-241 + core/io.py:146-170: every file below `path` that loads as an image (DICOM or Pillow), sorted."""
    import os

    found = []
    for root, _dirs, files in os.walk(str(path)):
        for name in files:
            full = os.path.join(root, name)
            if _is_dicom(full) or _is_image_file(full):
                found.append(full)
    return sorted(found)


class TemporaryZipDirectory:
    """core/io.py:87-117: a temporary directory holding the contents of a ZIP archive (path or binary stream)."""

    def __init__(self, zfile):
        import tempfile
        import zipfile

        self._tmp = tempfile.TemporaryDirectory()
        self.name = self._tmp.name
        with zipfile.ZipFile(zfile) as z:
            z.extractall(path=self.name)

    def __enter__(self) -> str:
        return self.name

    def __exit__(self, *exc) -> None:
        self._tmp.cleanup()


def load(path, **kwargs):
    """core/image.py:244-286.  ndarray -> ArrayImage, DICOM -> DicomImage, TIFF/PNG/JPG/BMP -> FileImage."""
    if isinstance(path, BaseImage):
        return path
    if _is_array(path):
        return ArrayImage(path, **kwargs)
    if _is_dicom(path):
        return DicomImage(path, **kwargs)
    if _is_image_file(path):
        return FileImage(path, **kwargs)
    raise TypeError(f"The argument `{path}` was not found to be a valid DICOM file, Image file, or array")


def equate_images(image1, image2):
    """core/image.py:169-220: crop the physically larger image and zoom the second one (cubic spline, scipy.ndimage.zoom semantics,
    on the device) so that both have the same pixel dimensions and DPI.  Returns (image1, image2) copies."""
    import copy

    image1, image2 = copy.deepcopy(image1), copy.deepcopy(image2)
    physical_height_diff = image1.physical_shape[0] - image2.physical_shape[0]
    img = image2 if physical_height_diff < 0 else image1
    pixel_height_diff = abs(int(round(-physical_height_diff * img.dpmm / 2)))
    if pixel_height_diff > 0:
        img.crop(pixel_height_diff, edges=("top", "bottom"))
    physical_width_diff = image1.physical_shape[1] - image2.physical_shape[1]
    img = image1 if physical_width_diff > 0 else image2
    pixel_width_diff = abs(int(round(physical_width_diff * img.dpmm / 2)))
    if pixel_width_diff > 0:
        img.crop(pixel_width_diff, edges=("left", "right"))
    zoom_factor = image1.shape[1] / image2.shape[1]
    image2_array = au.zoom(image2.as_type(float), zoom_factor)
    image2 = load(image2_array, dpi=image2.dpi * zoom_factor)
    return image1, image2


def load_multiples(image_file_list, method: str = "mean", stretch_each: bool = True, loader=None, **kwargs):
    """core/image.py:306-360: superimpose several images (files, arrays or image objects) into the first one.  With
    ``stretch_each`` every image is first stretched over the range of ``kwargs['dtype']`` ([0, 1] when absent; native ground /
    normalize), then the stack is reduced by 'mean' / 'max' / 'sum'.  The first image object carries the result and is flagged
    ``_raw_pixels`` (a later DICOM save converts instead of un-rescaling)."""
    reducers = {"mean": np.mean, "max": np.max, "sum": np.sum}
    if method not in reducers:
        raise ValueError("method must be one of 'mean', 'max', 'sum'")
    loader = loader or load
    images = [loader(item, **kwargs) for item in image_file_list]
    carrier = images[0]
    if any(im.shape != carrier.shape for im in images):
        raise ValueError("Images were not the same shape")
    planes = [au.stretcharray(im.array, fill_dtype=kwargs.get("dtype")) if stretch_each else im.array for im in images]
    carrier.array = reducers[method](np.stack(planes, axis=-1), axis=-1)
    carrier._raw_pixels = True
    return carrier


def _resaved(img):
    """What the reference obtains by writing a combined image to an in-memory DICOM and reading it back
    (DicomImage.save, core/image.py:1453-1489, then the constructor's rescale :363-389), without a DICOM writer:

    * values outside the stored dtype, and every ``_raw_pixels`` image, go through ``convert_to_dtype`` to the ORIGINAL stored
      dtype (full-range re-quantisation; otherwise the rescale is undone), then the plain ``astype``;
    * the reload applies RescaleSlope / RescaleIntercept and the PixelIntensityRelationshipSign flip of the file's own tags.

    Returns ``img`` with ``array`` / ``_stored`` / ``_stored_map`` replaced.  Array / file images are re-quantised to uint16."""
    a = np.asarray(img.array)
    if not isinstance(img, DicomImage):
        q = au.convert_to_dtype(a, np.uint16) if a.dtype.kind == "f" else a
        return ArrayImage(q, dpi=getattr(img, "_dpi", None) or img.dpi, sid=img.sid)
    if img._raw_pixels:
        un = a
    else:
        slope, intercept, flipped = img._stored_map
        un = a.max() + a.min() - a if flipped else a
        if img.metadata.get("RescaleSlope") is not None and img.metadata.get("RescaleIntercept") is not None:
            un = (un - intercept) / slope
    info = au.get_dtype_info(img._original_dtype)
    if un.max() > info.max or un.min() < info.min:
        import warnings

        warnings.warn("The pixel values of image were detected to be outside the range of the stored datatype and will be "
                      "normalized to fit it")
        un = au.convert_to_dtype(un, img._original_dtype)
    if img._raw_pixels:
        un = au.convert_to_dtype(un, img._original_dtype)
    stored = un.astype(img._original_dtype)
    img._raw_pixels = False
    img.array = _rescale_dicom_values(stored.copy(), img.metadata, False, None)
    slope, intercept = img.metadata.get("RescaleSlope"), img.metadata.get("RescaleIntercept")
    has = slope is not None and intercept is not None
    img._stored = stored
    img._stored_map = (float(slope) if has else 1.0, float(intercept) if has else 0.0,
                       img.metadata.get("PixelIntensityRelationshipSign") == -1)
    img._invert_pixels = None
    return img


def frame_u16(img, what: str = "GPU") -> np.ndarray:
    """The integer frame the device pipelines analyse, from an image object or an array.

    * uint16 is passed through, uint8 is widened, any other dtype whose values are integers in [0, 65535] is cast;
    * a float image that is still the DICOM rescale of its stored values (``stored * RescaleSlope + RescaleIntercept``, optionally
      flipped by ``PixelIntensityRelationshipSign``; core/image.py:363-389) is analysed on the STORED integers, order-flipped when
      the map is decreasing: every pipeline grounds / normalises / thresholds relative to the frame's own range, so a positive
      affine map changes sub-pixel results only by fp64 rounding (~1e-12 px), integer results not at all;
    * anything else (genuinely fractional pixel values) raises ``ValueError``.
    """
    a = img.array if isinstance(img, BaseImage) else np.asarray(img)
    if a.dtype == np.uint16:
        return a
    if a.dtype == np.uint8:
        return a.astype(np.uint16)
    if a.dtype.kind not in "fiu":
        raise TypeError(f"the {what} path takes numeric pixel data, got {a.dtype}")
    stored = getattr(img, "_stored", None)
    if stored is not None and stored.shape == a.shape and stored.dtype.kind == "u" and stored.dtype.itemsize <= 2:
        slope, intercept, flipped = img._stored_map
        if slope != 0:
            expect = stored.astype(np.float64) * slope + intercept if (slope, intercept) != (1.0, 0.0) else stored.astype(np.float64)
            if flipped:
                expect = expect.max() - expect + expect.min()
            if np.array_equal(a, expect):
                s16 = stored.astype(np.uint16)
                if flipped != (slope < 0):        # decreasing map of the stored values: exact modular order flip
                    s16 = (int(s16.max()) + int(s16.min()) - s16.astype(np.int64)).astype(np.uint16)
                return s16
    mn, mx = a.min(), a.max()
    if mn >= 0 and mx <= 65535 and np.array_equal(a, np.floor(a)):
        return a.astype(np.uint16)  # integer-valued pixels stored as another dtype (e.g. DICOM rescale 1.0 / 0.0)
    raise ValueError(f"the {what} path takes integer-valued pixel data in [0, 65535] (or a DICOM image whose array is still the "
                     "rescale of its stored values); got fractional / out-of-range values")


class BaseImage:
    """core/image.py:453-1102 (operators).  ``array`` is a host ndarray; operators rebind it to a fresh array."""

    array: np.ndarray

    def __init__(self, path):
        self.metrics = []
        self.metric_values = {}
        if isinstance(path, (str, Path)) and not osp.isfile(path):
            raise FileExistsError(f"File `{path}` does not exist. Verify the file path name.")
        elif isinstance(path, (str, Path)):
            self.path = path
            self.base_path = osp.basename(path)
        else:
            try:
                path.seek(0)
                self.path = str(Path(path.name))
            except AttributeError:
                self.path = ""

    # ------------------------------------------------------------------ geometry helpers (host)
    @property
    def center(self) -> Point:  # core/image.py:526-533
        return Point((self.shape[1] / 2) - 0.5, (self.shape[0] / 2) - 0.5)

    @property
    def physical_shape(self):  # core/image.py:535-538
        return self.shape[0] / self.dpmm, self.shape[1] / self.dpmm

    @property
    def shape(self):
        return self.array.shape

    @property
    def size(self):
        return self.array.size

    @property
    def ndim(self):
        return self.array.ndim

    @property
    def dtype(self):
        return self.array.dtype

    def sum(self):
        return self.array.sum()

    def ravel(self):
        return self.array.ravel()

    @property
    def flat(self):
        return self.array.flat

    def __len__(self):  # core/image.py:1098-1099
        return len(self.array)

    def __getitem__(self, item):  # core/image.py:1101-1102
        return self.array[item]

    def as_type(self, dtype):
        return self.array.astype(dtype)

    def gamma(self, comparison_image, doseTA: float = 1, distTA: float = 1, threshold: float = 0.1, ground: bool = True,
              normalize: bool = True) -> np.ndarray:
        """core/image.py:928-1017: Bakai gamma between this (reference) image and ``comparison_image`` -> float64 map (nan below the
        dose threshold).  The per-image preparation is the reference's (inversion check by histogram, ground, normalize: native
        operators); the Sobel gradient / hypot / division run in one fused kernel (csrc/gamma.cu)."""
        if not 0.0 <= threshold <= 1.0:
            raise ValueError("threshold must be between 0 and 1")
        if abs(self.dpi - comparison_image.dpi) > 0.1:
            raise AttributeError(f"The image DPIs to not match: {self.dpi:.2f} vs. {comparison_image.dpi:.2f}")
        same_x = abs(self.shape[1] - comparison_image.shape[1]) <= 1.1
        same_y = abs(self.shape[0] - comparison_image.shape[0]) <= 1.1
        if not (same_x and same_y) or self.shape != comparison_image.shape:
            raise AttributeError(f"The images are not the same size: {self.shape} vs. {comparison_image.shape}")

        def prepared(img) -> np.ndarray:
            tmp = ArrayImage(np.array(img.array, copy=True))
            tmp.check_inversion_by_histogram()
            if ground:
                tmp.ground()
            if normalize:
                tmp.normalize()
            if tmp.array.dtype.kind in "iub":     # ``array[below threshold] = nan`` on an integer array (core/image.py:1000)
                raise ValueError("cannot convert float NaN to integer")
            return np.ascontiguousarray(tmp.array, dtype=np.float64)

        ref, comp = prepared(self), prepared(comparison_image)
        ctx = nat.Context.default()
        with nat.Batch.upload(ctx, ref[None]) as rb, nat.Batch.upload(ctx, comp[None]) as cb:
            with rb._unary2(nat.lib().epid_gamma, cb, float(threshold * np.max(ref)), doseTA / 100.0, float(self.dpmm * distTA)) as out:
                return out.download()[0]

    def compute(self, metrics):
        """core/image.py:1022-1054: inject this image into the metric(s), calculate, store under a unique name."""
        from ..metrics.image import MetricBase

        if not hasattr(self, "metrics"):
            self.metrics, self.metric_values = [], {}
        metric_data = {}
        if isinstance(metrics, MetricBase):
            metrics = [metrics]
        key = None
        for metric in metrics:
            metric.inject_image(self)
            value = metric.context_calculate()
            self.metrics.append(metric)
            key = _uniquify(list(metric_data.keys()) + list(self.metric_values.keys()), metric.name)
            metric_data[key] = value
        self.metric_values |= metric_data
        if len(metrics) == 1:
            return metric_data[key]
        return metric_data

    # ------------------------------------------------------------------ operators
    def filter(self, size=0.05, kind: str = "median") -> None:  # core/image.py:695-712
        self.array = au.filter(self.array, size=size, kind=kind)

    def crop(self, pixels: int = 15, edges=("top", "bottom", "left", "right")) -> None:  # core/image.py:714-745
        if pixels < 0:
            raise ValueError("Pixels to remove must be a positive number")
        if pixels == 0:
            return
        if "top" in edges:
            self.array = self.array[pixels:, :]
        if "bottom" in edges:
            self.array = self.array[:-pixels, :]
        if "left" in edges:
            self.array = self.array[:, pixels:]
        if "right" in edges:
            self.array = self.array[:, :-pixels]
        if self.array.size == 0:
            raise ValueError("Too many pixels removed; array is empty. Pass a smaller crop value.")

    def flipud(self) -> None:
        self.array = np.flipud(self.array)

    def fliplr(self) -> None:
        self.array = np.fliplr(self.array)

    def invert(self) -> None:  # core/image.py:755-757
        self.array = au.invert(self.array)

    def bit_invert(self) -> None:  # core/image.py:759-761
        self.array = au.bit_invert(self.array)

    def roll(self, direction: str = "x", amount: int = 1) -> None:  # core/image.py:763-774
        axis = 1 if direction == "x" else 0
        self.array = np.roll(self.array, amount, axis=axis)

    def rotate(self, angle: float, mode: str = "edge", *args, **kwargs) -> None:  # core/image.py:780-783
        """Counter-clockwise rotation, scikit-image ``transform.rotate`` semantics with its defaults (bilinear, same shape; integer
        images are first scaled to [0, 1] like ``img_as_float``).  Other skimage keywords are not supported."""
        if args or kwargs:
            raise NotImplementedError("only rotate(angle, mode='edge' | 'constant') is implemented on the device")
        self.array = au.rotate(self.array, angle, mode=mode)

    def rot90(self, n: int = 1) -> None:
        self.array = np.rot90(self.array, n)

    def threshold(self, threshold: float, kind: str = "high") -> None:  # core/image.py:785-800
        self.array = au.threshold(self.array, threshold, kind)

    def as_binary(self, threshold):  # core/image.py:802-815
        return ArrayImage(au.binarize(self.array, threshold))

    def dist2edge_min(self, point) -> float:  # core/image.py:817-837
        if isinstance(point, tuple):
            point = Point(point)
        rows, cols = self.shape[0], self.shape[1]
        return min(rows - point.y, cols - point.x, point.y, point.x)

    def ground(self) -> float:  # core/image.py:839-853
        new, mn = au.ground_with_min(self.array)
        self.array = new
        return mn

    def normalize(self, norm_val=None) -> None:  # core/image.py:855-866
        if norm_val == "max":
            norm_val = None
        self.array = au.normalize(self.array, value=norm_val)

    def check_inversion(self, box_size: int = 20, position=(0.0, 0.0)) -> None:  # core/image.py:868-897
        a = self.array
        row_pos = max(int(position[0] * a.shape[0]), 1)
        col_pos = max(int(position[1] * a.shape[1]), 1)
        boxes = (a[row_pos : row_pos + box_size, col_pos : col_pos + box_size],
                 a[-row_pos - box_size : -row_pos, col_pos : col_pos + box_size],
                 a[row_pos : row_pos + box_size, -col_pos - box_size : -col_pos],
                 a[-row_pos - box_size : -row_pos, -col_pos - box_size : -col_pos])
        # 4 * box_size^2 corner pixels: a host reduction of a few hundred values; the frame mean is native
        avg = np.mean(boxes)
        if avg > au.frame_mean(a):
            self.invert()

    def check_inversion_by_histogram(self, percentiles=(5, 50, 95)) -> bool:  # core/image.py:899-926
        p_low, p_mid, p_high = au.percentile(self.array, percentiles)
        was_inverted = False
        if abs(p_mid - p_low) > abs(p_mid - p_high):
            was_inverted = True
            self.invert()
        return was_inverted


class ArrayImage(BaseImage):
    """core/image.py:1818-1867"""

    def __init__(self, array: np.ndarray, *, dpi: float | None = None, sid: float | None = None, dtype=None):
        self.metrics = []
        self.metric_values = {}
        if dtype is not None:
            self.array = np.array(array, dtype=dtype)
        else:
            self.array = array
        self._dpi = dpi
        self.sid = sid
        self.path = ""

    @property
    def dpmm(self) -> float | None:
        try:
            return self.dpi / MM_PER_INCH
        except Exception:
            return None

    @property
    def dpi(self) -> float | None:
        dpi = None
        if self._dpi is not None:
            dpi = self._dpi
            if self.sid is not None:
                dpi *= self.sid / 1000
        return dpi


class DicomImage(BaseImage):
    """core/image.py:1383-1580 with pylinac_b200.dicom instead of pydicom.  `path` may also be a ``dicom.Dataset`` already read
    (with ``pixel_array`` set, as DicomImageStack builds its slices): the image then views those pixels instead of copying them."""

    def __init__(self, path, *, dtype=None, dpi: float = None, sid: float = None, sad: float = 1000, raw_pixels: bool = False,
                 invert_pixels: bool | None = None):
        in_memory = isinstance(path, dicom.Dataset)
        super().__init__(path)
        self._sid = sid
        self._dpi = dpi
        self._sad = sad
        self.metadata = path if in_memory else dicom.dcmread(path)
        pix = self.metadata.pixel_array
        self._original_dtype = pix.dtype
        self._raw_pixels = raw_pixels
        self._invert_pixels = invert_pixels
        self.array = pix.astype(dtype) if dtype is not None else (pix if in_memory else pix.copy())
        self.array = _rescale_dicom_values(self.array, self.metadata, raw_pixels, invert_pixels)
        # the stored integers + the map that produced ``array`` from them (frame_u16 analyses the stored values when the
        # array is still that map of them)
        slope, intercept = self.metadata.get("RescaleSlope"), self.metadata.get("RescaleIntercept")
        has = (not raw_pixels) and slope is not None and intercept is not None
        sign = self.metadata.get("PixelIntensityRelationshipSign")
        flipped = (not raw_pixels) and bool(invert_pixels or (invert_pixels is None and sign == -1))
        self._stored = pix
        self._stored_map = (float(slope) if has else 1.0, float(intercept) if has else 0.0, flipped)

    @property
    def sid(self) -> float:
        try:
            return float(self.metadata.RTImageSID)
        except (AttributeError, ValueError, TypeError):
            return self._sid

    @property
    def sad(self) -> float:
        try:
            return float(self.metadata.RadiationMachineSAD)
        except (AttributeError, ValueError, TypeError):
            return self._sad

    @property
    def dpi(self) -> float:
        try:
            return self.dpmm * MM_PER_INCH
        except Exception:
            return self._dpi

    @property
    def dpmm(self) -> float:  # core/image.py:1534-1547
        dpmm = None
        for tag in ("PixelSpacing", "ImagePlanePixelSpacing"):
            mmpd = self.metadata.get(tag)
            if mmpd is not None:
                dpmm = 1 / mmpd[0]
                break
        if dpmm is not None and self.sid is not None:
            dpmm *= self.sid / self.sad
        elif dpmm is None and self._dpi is not None:
            dpmm = self._dpi / MM_PER_INCH
        return dpmm

    @property
    def cax(self) -> Point:  # core/image.py:1550-1580
        try:
            mag_factor = self.sid / self.sad
            t = self.metadata.XRayImageReceptorTranslation
            return Point(self.center.x - t[0] * self.dpmm / mag_factor, self.center.y + t[1] * self.dpmm / mag_factor)
        except (AttributeError, ValueError, TypeError, KeyError):
            return self.center


def _rescale_dicom_values(unscaled, metadata, raw_pixels, invert_pixels):
    """core/image.py:363-389 (pydicom apply_rescale: only when RescaleSlope/Intercept are present)."""
    if raw_pixels:
        return unscaled
    slope, intercept = metadata.get("RescaleSlope"), metadata.get("RescaleIntercept")
    scaled = unscaled
    if slope is not None and intercept is not None:
        # pydicom.pixels.apply_rescale: arr * slope + intercept -> float64 (kept integral dtype when the map is identity)
        if not (float(slope) == 1.0 and float(intercept) == 0.0):
            scaled = unscaled.astype(np.float64) * float(slope) + float(intercept)
        else:
            scaled = unscaled.astype(np.float64)
    sign = metadata.get("PixelIntensityRelationshipSign")
    if invert_pixels or (invert_pixels is None and sign == -1):
        scaled = scaled.max() - scaled + scaled.min()
    return scaled


class FileImage(BaseImage):
    """core/image.py:1733-1812: TIFF / PNG / JPG / BMP through Pillow (host-side ingest)."""

    def __init__(self, path, *, dpi: float | None = None, sid: float | None = None, dtype=None):
        from PIL import Image as pImage
        from PIL.TiffTags import TAGS

        super().__init__(path)
        pil_image = pImage.open(path)
        if len(pil_image.getbands()) > 1:
            pil_image = pil_image.convert("I")  # multi-channel -> int32 (core/image.py:1770-1774)
        self.info = pil_image.info
        try:
            self.tags = {TAGS[key]: pil_image.tag_v2[key] for key in pil_image.tag_v2}
        except AttributeError:
            pass
        self.array = np.array(pil_image, dtype=dtype)
        self._dpi = dpi
        self.sid = sid

    @property
    def dpi(self) -> float | None:  # core/image.py:1784-1803
        dpi = None
        for key in ("dpi", "resolution"):
            dpi = self.info.get(key)
            if dpi is not None:
                dpi = float(dpi[0])
                if dpi < 3 and not self._dpi:
                    raise ValueError(f"The DPI setting is abnormal or nonsensical. Got resolution of {dpi}. Pass in the dpi manually.")
                if dpi < 3:
                    dpi = None
                break
        if dpi is None:
            dpi = self._dpi
        if self.sid is not None and dpi is not None:
            dpi *= self.sid / 1000
        return dpi

    @property
    def dpmm(self) -> float | None:
        try:
            return self.dpi / MM_PER_INCH
        except TypeError:
            return None


class LinacDicomImage(DicomImage):
    """core/image.py:1583-1730: gantry / collimator / couch angles from tags or overrides."""

    def __init__(self, path, use_filenames: bool = False, axes_precision: int | None = None, missing_axis_value=0, **kwargs):
        self._axis_overrides = {}
        for axis in ("gantry", "coll", "couch"):
            if axis in kwargs:
                self._axis_overrides[axis] = kwargs.pop(axis)
        self._axes_precision = axes_precision
        self._missing_axis_value = missing_axis_value
        self._use_filenames = use_filenames
        super().__init__(path, **kwargs)

    _AXIS_NAMES = {"gantry": "Gantry", "coll": "Coll", "couch": "Couch"}

    def _axis(self, key, tag):
        return linac_axis_value(key, self._axis_overrides.get(key), self.path, self.metadata.get(tag), use_filenames=self._use_filenames,
                                missing_axis_value=self._missing_axis_value, axes_precision=self._axes_precision)

    @property
    def gantry_angle(self) -> float:
        return self._axis("gantry", "GantryAngle")

    @property
    def collimator_angle(self) -> float:
        return self._axis("coll", "BeamLimitingDeviceAngle")

    @property
    def couch_angle(self) -> float:
        return self._axis("couch", "PatientSupportAngle")


def linac_axis_value(key: str, override, path, tag_value, *, use_filenames: bool, missing_axis_value, axes_precision):
    """_get_axis_value (core/image.py:1655-1730) of axis `key` ('gantry' / 'coll' / 'couch'): explicit value, else `<axis><number>`
    in the file name when use_filenames (keyword absent -> missing_axis_value, the tags are not consulted), else the DICOM tag value,
    else missing_axis_value."""
    import re

    name = LinacDicomImage._AXIS_NAMES[key]
    if override is not None:
        v = override
    elif use_filenames:
        filename = osp.basename(str(path)).lower()
        if name.lower() not in filename:
            if missing_axis_value == "raise":
                raise ValueError(f"{name} axis value was not found in the filename and `missing_axis_value` was `raise`. "
                                 "Either provide an axis value or pass a numerical value for `missing_axis_value`.")
            v = missing_axis_value
        else:
            m = re.search(rf"(?<={name.lower()})\d+", filename)
            if m is None:
                raise ValueError(f"The filename contains '{name}' but could not read a number following it. "
                                 f"Use the format '...{name}<#>...'")
            v = float(m.group())
    else:
        v = tag_value
        if v is None:
            if missing_axis_value == "raise":
                raise ValueError(f"Axis {key} was not found in the DICOM tags")
            v = missing_axis_value
    v = float(v)
    if axes_precision is not None:
        v = round(v, axes_precision)
    return v % 360 if v >= 360 else v


def _image_header(path):
    """LazyDicomImageStack._get_path_metadatas (core/image.py:1952-1966) for one file: its header when its SOP Class UID names an
    image storage class; None for a file that does not parse as DICOM, has no SOP Class UID or is not an image."""
    try:
        ds = dicom.read_header(path)
        uid = ds.SOPClassUID
    except OSError:
        raise
    except Exception:
        return None
    return ds if uid in dicom.IMAGE_STORAGE_UIDS else None


class DicomImageStack:
    """core/image.py:1873-2210 (LazyDicomImageStack.__init__ + DicomImageStack.__init__): the image files of a folder (searched
    recursively; a list or tuple of paths is taken as given), filtered to the most common SeriesInstanceUID and sorted by the last
    ImagePositionPatient coordinate.  Headers are parsed on a thread pool without touching pixel data, then every slice's pixels are
    read in sorted order into one [n, rows, cols] page-locked array, ``volume``; ``images[i]`` is a DicomImage viewing
    ``volume[i]`` (``dtype`` / ``raw_pixels`` applied as DicomImage applies them)."""

    def __init__(self, folder, dtype=None, min_number: int = 39, check_uid: bool = True, raw_pixels: bool = False):
        from collections import Counter
        from concurrent.futures import ThreadPoolExecutor

        self.dtype = dtype
        paths = []
        if isinstance(folder, (list, tuple)):
            paths = [str(p) for p in folder]
        elif osp.isdir(folder):
            for pdir, _sdir, files in os.walk(folder):
                for file in files:
                    paths.append(osp.join(pdir, file))
        with ThreadPoolExecutor(max(1, min(8, len(paths)))) as pool:
            headers = list(pool.map(_image_header, paths))
        metadatas = [h for h in headers if h is not None]
        paths = [p for p, h in zip(paths, headers) if h is not None]
        if len(paths) < 1:
            raise FileNotFoundError(f"No files were found in the specified location: {folder}")
        if check_uid:
            most_common_uid = Counter(m.SeriesInstanceUID for m in metadatas).most_common(1)[0]
            if most_common_uid[1] < min_number:
                raise ValueError("The minimum number images from the same study were not found")
            keep = [k for k, m in enumerate(metadatas) if m.SeriesInstanceUID == most_common_uid[0]]
            metadatas, paths = [metadatas[k] for k in keep], [paths[k] for k in keep]
        order = np.argsort([m.ImagePositionPatient[-1] for m in metadatas])
        self.metadatas = [metadatas[i] for i in order]
        self._image_path_keys = [paths[i] for i in order]
        h0 = self.metadatas[0]
        shape = (len(self.metadatas), int(h0["Rows"]), int(h0["Columns"]))
        try:
            volume = nat.pinned_empty(shape, h0["PixelDtype"])
        except nat.NativeError:      # no CUDA device: pageable host memory (only the H2D copy is slower)
            volume = None
        self.volume, _ = dicom.read_frames(self._image_path_keys, out=volume, headers=self.metadatas)
        for m, pixels in zip(self.metadatas, self.volume):
            m.pixel_array = pixels
        self.images = [DicomImage(m, dtype=dtype, raw_pixels=raw_pixels) for m in self.metadatas]

    @classmethod
    def from_zip(cls, zip_path, dtype=None, **kwargs):
        """core/image.py:2167-2180"""
        with TemporaryZipDirectory(zip_path) as tmpzip:
            return cls(tmpzip, dtype, **kwargs)

    @property
    def metadata(self):
        """The metadata of the first (sorted) slice."""
        return self[0].metadata

    @property
    def slice_spacing(self) -> float:
        """core/image.py:1983-1989: distance between the first two slices."""
        return np.abs(self.metadatas[0].ImagePositionPatient[-1] - self.metadatas[1].ImagePositionPatient[-1])

    def __getitem__(self, item) -> DicomImage:
        return self.images[item]

    def __len__(self):
        return len(self.images)


class NMImageStack:
    """core/image.py:2216-2249: the N frames of one nuclear medicine file, each a DicomImage holding the stored frame as is.
    Every frame is read by one ``dicom.read_nm_frames`` pass into page-locked memory (pageable without a CUDA device)."""

    def __init__(self, path):
        self.path = path
        self.metadata = dicom.read_header(path)
        if self.metadata.get("Modality") != "NM":
            raise TypeError("The file is not a NM image")
        shape = (int(self.metadata.get("NumberOfFrames", 1) or 1), int(self.metadata["Rows"]), int(self.metadata["Columns"]))
        try:
            out = nat.pinned_empty(shape, self.metadata["PixelDtype"])
        except nat.NativeError:      # no CUDA device: pageable host memory (only the H2D copy is slower)
            out = None
        self._pixels, _ = dicom.read_nm_frames([path], out=out)
        self.frames = []
        for pixels in self._pixels:
            ds = dicom.Dataset(self.metadata)
            ds.pixel_array = pixels
            img = DicomImage(ds)
            img.array = pixels           # the reference assigns the stored frame, without the rescale DicomImage applies
            self.frames.append(img)

    def as_3d_array(self) -> np.ndarray:
        """the frames stacked into one [n, h, w] array (a copy)"""
        return np.stack([i.array for i in self.frames], axis=0)

    def __len__(self):
        return len(self.frames)


class XIM(BaseImage):
    """core/image.py:1105-1318: a Varian .xim image (TrueBeam / Halcyon EPID and kV, IsoCal and MPC exports).  The header and
    property walk is the reference's (pylinac_b200.xim); the compressed pixels are decoded on the GPU (csrc/xim.cu) through the
    same entry point as batched ingest, with n = 1.  Export (save_as / as_dicom) is not provided."""

    array: np.ndarray
    properties: dict

    def __init__(self, file_path: str | Path, read_pixels: bool = True):
        from .. import xim

        super().__init__(path=file_path)
        hd = xim.walk(self.path, read_pixels=read_pixels)
        if hd.compression and read_pixels:
            self.array = xim.decode_file(hd)
            if hd.trailer_error is not None:
                raise hd.trailer_error
        for name in ("format_id", "format_version", "img_width_px", "img_height_px", "bits_per_pixel", "bytes_per_pixel",
                     "compression", "num_hist_bins", "histogram", "num_properties", "properties"):
            setattr(self, name, getattr(hd, name))
        if hd.compression:
            self.lookup_table = hd.lookup_table
        else:
            self.pixel_buffer = hd.pixel_buffer

    @property
    def dpmm(self) -> float:  # core/image.py:1311-1318
        """The dots/mm value of the XIM images. The value appears to be in cm in the file."""
        if self.properties["PixelWidth"] != self.properties["PixelHeight"]:
            raise ValueError("The XIM image does not have the same pixel height and width")
        return 1 / (10 * self.properties["PixelHeight"])
