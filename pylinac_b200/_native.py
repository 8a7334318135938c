"""ctypes binding of ``libepid.so`` (the C-ABI declared in ``include/epid.h``).

This is the only module that touches the native library.  There is NO CPU fallback: if the shared
library is missing, or no CUDA device is visible, the compute entry points raise.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import subprocess
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("EPID_LIB") or os.path.join(_HERE, "libepid.so")      # EPID_LIB: kernel-variant experiments (tools/)

EPID_OK = 0
ERR_NO_DEVICE, ERR_CUDA, ERR_INVALID, ERR_UNSUPPORTED, ERR_NOMEM, ERR_NCCL = -1, -2, -3, -4, -5, -6

U8, U16, I32, F32, F64, I16, I64 = 0, 1, 2, 3, 4, 5, 6
_NP2DT = {np.dtype(np.uint8): U8, np.dtype(np.uint16): U16, np.dtype(np.int32): I32, np.dtype(np.float32): F32,
          np.dtype(np.float64): F64, np.dtype(np.int16): I16, np.dtype(np.int64): I64}
_DT2NP = {v: k for k, v in _NP2DT.items()}

OPT_PF_EXACT_ONLY = 1
OPT_PF_WIN2 = 3
OPT_STATS_EXACT = 7
CTR_PF_FALLBACKS = 1
CTR_PF_REDONE_FRAMES = 2
CTR_PF_EXACT_FRAMES = 3
CTR_STATS_UNCERTIFIED = 4
PF_MAX_PICKETS = 32
PF_MAX_LEAVES = 160


class NativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libepid error {code}: {msg}")
        self.code = code
        self.msg = msg


class NoDeviceError(NativeError):
    pass


PEAKS_ALL = -(2 ** 31)   # EPID_PEAKS_ALL: max_number=None


class PeakParams(C.Structure):
    _fields_ = [("threshold", C.c_double), ("peak_separation", C.c_double), ("max_number", C.c_int32),
                ("fwxm_height", C.c_double), ("min_width", C.c_double), ("search_lo", C.c_double),
                ("search_hi", C.c_double), ("peak_sort", C.c_int32), ("required_prominence", C.c_double)]


class PFParams(C.Structure):
    _fields_ = [("dpmm", C.c_double), ("crop_px", C.c_int32), ("filter_size", C.c_int32), ("tolerance", C.c_double),
                ("action_tolerance", C.c_double), ("num_pickets", C.c_int32), ("sag_px", C.c_int32),
                ("orientation", C.c_int32), ("invert", C.c_int32), ("leaf_analysis_width_ratio", C.c_double),
                ("picket_spacing", C.c_double), ("height_threshold", C.c_double), ("edge_threshold", C.c_double),
                ("peak_sort", C.c_int32), ("required_prominence", C.c_double), ("separate_leaves", C.c_int32),
                ("nominal_gap_mm", C.c_double), ("has_cax_override", C.c_int32), ("cax_x_px", C.c_double),
                ("cax_y_px", C.c_double), ("n_leaves", C.c_int32), ("leaf_center_mm", C.c_double * PF_MAX_LEAVES),
                ("leaf_width_mm", C.c_double * PF_MAX_LEAVES), ("leaf_num", C.c_int32 * PF_MAX_LEAVES)]


PF_SUMMARY_DTYPE = np.dtype([
    ("status", "<i4"), ("orientation", "<i4"), ("noise_median_passes", "<i4"), ("corner_inverted", "<i4"),
    ("height", "<i4"), ("width", "<i4"), ("n_pickets", "<i4"), ("n_meas", "<i4"), ("n_leaves_removed", "<i4"),
    ("passed", "<i4"), ("max_error_picket", "<i4"), ("max_error_leaf", "<i4"), ("max_error_bank", "<i4"),
    ("n_failed", "<i4"), ("picket_spacing_px", "<f8"), ("percent_passing", "<f8"), ("max_error_mm", "<f8"),
    ("abs_median_error_mm", "<f8"), ("mean_picket_spacing_mm", "<f8"), ("mlc_skew", "<f8"), ("cax_px", "<f8"),
    ("picket_idx", "<i4", (PF_MAX_PICKETS,)), ("picket_val", "<f8", (PF_MAX_PICKETS,)),
    ("fit_slope", "<f8", (PF_MAX_PICKETS,)), ("fit_intercept", "<f8", (PF_MAX_PICKETS,)),
    ("offsets_from_cax_mm", "<f8", (PF_MAX_PICKETS,)), ("picket_width_max", "<f8", (PF_MAX_PICKETS,)),
    ("picket_width_mean", "<f8", (PF_MAX_PICKETS,)), ("picket_width_median", "<f8", (PF_MAX_PICKETS,)),
    ("picket_width_min", "<f8", (PF_MAX_PICKETS,))], align=True)
PF_MEAS_DTYPE = np.dtype([("leaf_num", "<i4"), ("picket", "<i4"), ("passed", "<i4", (2,)), ("position", "<f8", (2,)),
                          ("error", "<f8", (2,)), ("width_mm", "<f8")], align=True)

STAR_MAX_PEAKS = 64


class StarParams(C.Structure):
    _fields_ = [("dpmm", C.c_double), ("radius", C.c_double), ("min_peak_height", C.c_double), ("max_wobble_diameter", C.c_double),
                ("tolerance", C.c_double), ("has_start_point", C.c_int32), ("start_x", C.c_double), ("start_y", C.c_double),
                ("fwhm", C.c_int32), ("recursive", C.c_int32), ("invert", C.c_int32)]


STAR_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("hist_inverted", "<i4"), ("start_x", "<i4"), ("start_y", "<i4"), ("local_max", "<f8"),
    ("iterations", "<i4"), ("profile_len", "<i4"), ("radius_px", "<f8"), ("n_peaks", "<i4"), ("n_lines", "<i4"),
    ("peak_idx", "<i4", (STAR_MAX_PEAKS,)), ("peak_x", "<f8", (STAR_MAX_PEAKS,)), ("peak_y", "<f8", (STAR_MAX_PEAKS,)),
    ("wobble_x", "<f8"), ("wobble_y", "<f8"), ("wobble_radius_px", "<f8"), ("wobble_radius_mm", "<f8"),
    ("angles", "<f8", (STAR_MAX_PEAKS // 2,)), ("passed", "<i4"), ("pad", "<i4")], align=True)


class FieldParams(C.Structure):
    _fields_ = [("dpmm", C.c_double), ("protocol", C.c_int32), ("centering", C.c_int32), ("vert_position", C.c_double),
                ("horiz_position", C.c_double), ("vert_width", C.c_double), ("horiz_width", C.c_double),
                ("in_field_ratio", C.c_double), ("slope_exclusion_ratio", C.c_double), ("invert", C.c_int32),
                ("penumbra_lower", C.c_double), ("penumbra_upper", C.c_double), ("interpolation", C.c_int32),
                ("interpolation_resolution_mm", C.c_double), ("ground", C.c_int32), ("normalization", C.c_int32),
                ("edge", C.c_int32), ("edge_smoothing_ratio", C.c_double)]


FIELD_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("hist_inverted", "<i4"), ("strip_rows", "<i4", (2,)), ("strip_cols", "<i4", (2,)), ("profile_len", "<i4", (2,)),
    ("top_penumbra_mm", "<f8"), ("bottom_penumbra_mm", "<f8"), ("left_penumbra_mm", "<f8"), ("right_penumbra_mm", "<f8"),
    ("geometric_center_index_x_y", "<f8", (2,)), ("beam_center_index_x_y", "<f8", (2,)),
    ("field_size_vertical_mm", "<f8"), ("field_size_horizontal_mm", "<f8"),
    ("beam_center_to_top_mm", "<f8"), ("beam_center_to_bottom_mm", "<f8"), ("beam_center_to_left_mm", "<f8"),
    ("beam_center_to_right_mm", "<f8"), ("cax_to_top_mm", "<f8"), ("cax_to_bottom_mm", "<f8"), ("cax_to_left_mm", "<f8"),
    ("cax_to_right_mm", "<f8"), ("top_position_index_x_y", "<f8", (2,)),
    ("top_horizontal_distance_from_cax_mm", "<f8"), ("top_vertical_distance_from_cax_mm", "<f8"),
    ("top_horizontal_distance_from_beam_center_mm", "<f8"), ("top_vertical_distance_from_beam_center_mm", "<f8"),
    ("left_slope_percent_mm", "<f8"), ("right_slope_percent_mm", "<f8"), ("top_slope_percent_mm", "<f8"),
    ("bottom_slope_percent_mm", "<f8"), ("symmetry_horizontal", "<f8"), ("symmetry_vertical", "<f8"),
    ("flatness_horizontal", "<f8"), ("flatness_vertical", "<f8")], align=True)


class SpParams(C.Structure):
    _fields_ = [("dpmm", C.c_double), ("interpolation", C.c_int32), ("interpolation_resolution_mm", C.c_double),
                ("interpolation_factor", C.c_double), ("ground", C.c_int32), ("normalization", C.c_int32), ("edge", C.c_int32),
                ("centering", C.c_int32), ("edge_smoothing_ratio", C.c_double), ("x_start", C.c_double), ("x_stop", C.c_double),
                ("edge_left", C.c_double), ("edge_right", C.c_double)]


SP_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("n", "<i4"), ("x_start", "<f8"), ("x_stop", "<f8"), ("values_max", "<f8"),
    ("geometric_center_index", "<f8"), ("geometric_center_value", "<f8"),
    ("beam_ok", "<i4"), ("fwxm_ok", "<i4"), ("infl_ok", "<i4"), ("pen_ok", "<i4"), ("fd_ok", "<i4"), ("fd_field_values_n", "<i4"),
    ("beam_center_index", "<f8"), ("beam_center_value_at_rounded", "<f8"),
    ("fwxm_left", "<f8"), ("fwxm_right", "<f8"), ("fwxm_center_value_at_rounded", "<f8"), ("fwxm_left_value_at_rounded", "<f8"),
    ("fwxm_right_value_at_rounded", "<f8"),
    ("infl_left", "<f8"), ("infl_right", "<f8"), ("infl_left_value_exact", "<f8"), ("infl_right_value_exact", "<f8"),
    ("infl_left_value_rounded", "<f8"), ("infl_right_value_rounded", "<f8"),
    ("pen_left_lower", "<f8"), ("pen_left_upper", "<f8"), ("pen_right_lower", "<f8"), ("pen_right_upper", "<f8"),
    ("fd_width", "<f8"), ("fd_beam_center", "<f8"), ("fd_cax", "<f8"), ("fd_left", "<f8"), ("fd_right", "<f8"),
    ("fd_inner_left", "<f8"), ("fd_inner_right", "<f8"), ("fd_left_slope", "<f8"), ("fd_left_intercept", "<f8"),
    ("fd_right_slope", "<f8"), ("fd_right_intercept", "<f8"), ("fd_top_index", "<f8"), ("fd_top_value", "<f8"),
    ("fd_top_params", "<f8", (3,)), ("fd_beam_center_value", "<f8"), ("fd_cax_value", "<f8"), ("fd_left_value", "<f8"),
    ("fd_right_value", "<f8")], align=True)


class WlParams(C.Structure):
    _fields_ = [("dpmm", C.c_double), ("bb_size_mm", C.c_double), ("low_density_bb", C.c_int32), ("open_field", C.c_int32),
                ("bb_proximity_mm", C.c_double)]


(WL_OK, WL_NO_BB, WL_MISMATCH, WL_NO_FIELD, WL_CAPACITY, WL_FLAT_IMAGE) = range(6)
WL_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("inverted", "<i4"), ("crop_px", "<i4"), ("height", "<i4"), ("width", "<i4"), ("n_bbs", "<i4"),
    ("threshold_passes", "<i4"), ("pad", "<i4"), ("bb_x", "<f8"), ("bb_y", "<f8"), ("field_x", "<f8"), ("field_y", "<f8"),
    ("epid_x", "<f8"), ("epid_y", "<f8"), ("cax2bb_x", "<f8"), ("cax2bb_y", "<f8"), ("cax2bb_distance", "<f8"),
    ("cax2epid_x", "<f8"), ("cax2epid_y", "<f8"), ("cax2epid_distance", "<f8")], align=True)
DISK_MAX = 8


class DiskParams(C.Structure):
    """epid_disk_params (include/epid.h)"""

    _fields_ = [("dpmm", C.c_double), ("expected_x", C.c_double), ("expected_y", C.c_double), ("window_w", C.c_double),
                ("window_h", C.c_double), ("radius_mm", C.c_double), ("tolerance_mm", C.c_double), ("min_separation_px", C.c_double),
                ("invert", C.c_int32), ("max_number", C.c_int32), ("conditions", C.c_int32), ("pad", C.c_int32)]


_D = (DISK_MAX,)
DISK_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("n_points", "<i4"), ("n_regions", "<i4"), ("passes", "<i4"), ("left", "<i4"), ("top", "<i4"), ("x", "<f8", _D),
    ("y", "<f8", _D), ("r_area", "<f8", _D), ("r_filled_area", "<f8", _D), ("r_perimeter", "<f8", _D), ("r_convex_area", "<f8", _D),
    ("r_centroid_y", "<f8", _D), ("r_centroid_x", "<f8", _D), ("r_wcentroid_y", "<f8", _D), ("r_wcentroid_x", "<f8", _D),
    ("r_bbox", "<i4", (DISK_MAX, 4))], align=True)
_lib = None
_lock = threading.Lock()


def build(force: bool = False) -> str:
    """Compile libepid.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    src = os.path.join(_HERE, "csrc")
    if force:
        subprocess.run(["make", "-C", src, "clean"], check=True, stdout=subprocess.DEVNULL)
    subprocess.run(["make", "-C", src, "-j8"], check=True, stdout=subprocess.DEVNULL)
    return LIB_PATH


VMAT_MAX_SEG = 16


class VmatParams(C.Structure):
    _fields_ = [("ground", C.c_int32), ("check_inversion", C.c_int32), ("invert_image_order", C.c_int32), ("nseg", C.c_int32),
                ("dpmm", C.c_double), ("tolerance_percent", C.c_double), ("seg_w_mm", C.c_double), ("seg_h_mm", C.c_double),
                ("offset_mm", C.c_double * VMAT_MAX_SEG)]


_S = (VMAT_MAX_SEG,)
VMAT_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("open_is_first", "<i4"), ("inverted", "<i4", (2,)), ("center_warning", "<i4"), ("passed", "<i4"), ("nseg", "<i4"),
    ("pad_", "<i4"), ("x_field_center", "<f8"), ("profile_center_idx", "<f8", (2,)), ("field_len", "<f8", (2,)), ("field_std", "<f8", (2,)),
    ("r_corr", "<f8", _S), ("r_dev", "<f8", _S), ("stdev", "<f8", _S), ("center_x", "<f8", _S), ("center_y", "<f8", _S), ("npix", "<f8", _S),
    ("seg_passed", "<i4", _S), ("max_r_deviation", "<f8"), ("avg_abs_r_deviation", "<f8"), ("avg_r_deviation", "<f8")], align=True)



LR_MAX_BB = 5
LR_SCALING = 5


class LrParams(C.Structure):
    """epid_lr_params (include/epid.h)"""

    _fields_ = [("dpmm", C.c_double), ("fwxm", C.c_double), ("bb_edge_threshold_mm", C.c_double), ("bb_size_mm", C.c_double),
                ("bb_box_mm", C.c_double), ("strip_width_mm", C.c_double), ("quasar_offset_mm", C.c_double),
                ("bb_mm", C.c_double * (2 * LR_MAX_BB)), ("bb15_mm", C.c_double * (2 * LR_MAX_BB)), ("nbb", C.c_int32),
                ("set_mode", C.c_int32), ("normalize", C.c_int32), ("invert", C.c_int32), ("clahe_kernel", C.c_int32),
                ("scaling", C.c_int32)]


LR_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("inverted", "<i4"), ("large_set", "<i4"), ("near_edge_mask", "<i4"), ("failed_bb", "<i4"), ("n_found", "<i4"),
    ("n_scaling", "<i4"), ("pad", "<i4"), ("field_center_x", "<f8"), ("field_center_y", "<f8"), ("field_width_x_mm", "<f8"),
    ("field_width_y_mm", "<f8"), ("bb_x", "<f8", (LR_MAX_BB,)), ("bb_y", "<f8", (LR_MAX_BB,)), ("scaling_x", "<f8", (LR_SCALING,)),
    ("scaling_y", "<f8", (LR_SCALING,))], align=True)


class LocateParams(C.Structure):
    _fields_ = [("mode", C.c_int32), ("invert", C.c_int32), ("sample_kind", C.c_int32), ("conditions", C.c_int32), ("dpmm", C.c_double),
                ("radius_mm", C.c_double), ("tolerance_mm", C.c_double), ("field_width_mm", C.c_double), ("field_height_mm", C.c_double),
                ("field_tolerance_mm", C.c_double), ("bb_size_mm", C.c_double), ("rad_size_mm", C.c_double)]


NM_OK, NM_NO_COMPONENT = 0, 1

NM_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("longest", "<i4"), ("erosion", "<i4", (2,)), ("n_fov", "<i4", (2,)), ("max_index", "<i4", (2,)),
    ("min_index", "<i4", (2,)), ("du_count", "<i4", (4,)), ("du_index", "<i4", (4,)), ("threshold", "<f8"), ("iu", "<f8", (2,)),
    ("du_max", "<f8", (4,))], align=True)


NT_OK, NT_NO_COMPONENT = 0, 1

NT_SLICE_DTYPE = np.dtype([
    ("status", "<i4"), ("longest", "<i4"), ("erosion", "<i4"), ("area", "<i4"), ("max", "<i4"), ("min", "<i4"), ("sum", "<u8"),
    ("centroid_row", "<f8"), ("centroid_col", "<f8"), ("uniformity", "<f8"), ("value", "<f8")], align=True)

NT_SPHERE_IN_DTYPE = np.dtype([("x0", "<f8", (3,)), ("lb", "<f8", (3,)), ("ub", "<f8", (3,)), ("r2", "<f8"), ("baseline", "<f8"),
                               ("volume", "<i4"), ("pad", "<i4")], align=True)

NT_SPHERE_DTYPE = np.dtype([
    ("nfev", "<i4"), ("nit", "<i4"), ("status", "<i4"), ("n_empty", "<i4"), ("count", "<i4"), ("min", "<i4"), ("sum", "<u8"),
    ("x", "<f8", (3,)), ("fun", "<f8")], align=True)


TU_RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("longest", "<i4"), ("erosion", "<i4", (3,)), ("n_fov", "<i4", (3,)), ("max_index", "<i4", (3,)),
    ("min_index", "<i4", (3,)), ("du_count", "<i4", (6,)), ("du_index", "<i4", (6,)), ("center_count", "<i4"), ("ring_count", "<i4"),
    ("threshold", "<f8"), ("iu", "<f8", (3,)), ("du_max", "<f8", (6,)), ("center_sum", "<f8"), ("ring_sum", "<f8")], align=True)


CT_OK, CT_NO_EDGES, CT_NO_REGIONS, CT_WRONG_SIZE = 0, 1, 2, 3

CT_SLICE_DTYPE = np.dtype([("status", "<i4"), ("n_regions", "<i4"), ("label", "<i4"), ("area", "<i4"), ("centroid_row", "<f8"),
                           ("centroid_col", "<f8"), ("max_edge", "<f8"), ("threshold", "<f8")], align=True)

CT_REGION_DTYPE = np.dtype([("label", "<i4"), ("first", "<i4"), ("area", "<i4"), ("filled_area", "<i4"), ("bbox", "<i4", (4,)),
                            ("sum_r", "<u8"), ("sum_c", "<u8"), ("m_rr", "<u8"), ("m_cc", "<u8"), ("m_rc", "<u8")], align=True)


REGION_DTYPE = np.dtype([("threshold_index", "<i4"), ("label_root", "<i4"), ("bbox", "<i4", (4,)), ("area", "<f8"), ("area_filled", "<f8"),
                         ("perimeter", "<f8"), ("equivalent_diameter", "<f8"), ("centroid_y", "<f8"), ("centroid_x", "<f8"),
                         ("wcentroid_y", "<f8"), ("wcentroid_x", "<f8")], align=True)

_P = C.c_void_p
_SIGNATURES = {
    "epid_device_count": [C.POINTER(C.c_int32)],
    "epid_ctx_create": [C.c_int32, C.POINTER(_P)],
    "epid_ctx_destroy": [_P],
    "epid_sync": [_P],
    "epid_device_info": [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_size_t)],
    "epid_device_pci_bus_id": [C.c_int32, C.c_char_p, C.c_int32],
    "epid_launch_count": [_P, C.POINTER(C.c_int64)],
    "epid_version": [],
    "epid_set_option": [_P, C.c_int32, C.c_int64],
    "epid_get_counter": [_P, C.c_int32, C.POINTER(C.c_int64)],
    "epid_host_alloc": [C.c_size_t, C.POINTER(_P)],
    "epid_host_free": [_P],
    "epid_batch_upload": [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)],
    "epid_batch_alloc": [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)],
    "epid_batch_download": [_P, _P],
    "epid_batch_write": [_P, _P],
    "epid_batch_free": [_P],
    "epid_batch_shape": [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)],
    "epid_batch_device_ptr": [_P, C.POINTER(_P)],
    "epid_frame_stats": [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, _P, _P, _P],
    "epid_frame_histogram": [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P],
    "epid_invert": [_P, _P, C.POINTER(_P)],
    "epid_bit_invert": [_P, _P, C.POINTER(_P)],
    "epid_ground": [_P, _P, C.c_double, C.POINTER(_P), _P],
    "epid_normalize": [_P, _P, C.c_int32, C.c_double, C.POINTER(_P)],
    "epid_threshold": [_P, _P, C.c_double, C.c_int32, C.POINTER(_P)],
    "epid_binarize": [_P, _P, C.c_double, C.POINTER(_P)],
    "epid_median_filter": [_P, _P, C.c_int32, C.POINTER(_P)],
    "epid_gaussian_filter": [_P, _P, C.c_double, C.POINTER(_P)],
    "epid_correlate1d_passes": [_P, _P, _P, C.c_int32, C.c_int32, C.POINTER(_P)],
    "epid_sobel": [_P, _P, C.c_int32, C.POINTER(_P)],
    "epid_find_peaks": [_P, _P, C.c_int32, C.POINTER(PeakParams), C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                        C.POINTER(C.c_int32)],
    "epid_pf_analyze": [_P, _P, C.POINTER(PFParams), _P, _P, C.c_int32],
    "epid_pf_analyze_host": [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(PFParams), _P, _P, C.c_int32],
    "epid_pf_bench": [_P, _P, C.POINTER(PFParams), C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float),
                      C.POINTER(C.c_int64)],
    "epid_pf_bench_stages": [_P, _P, C.POINTER(PFParams), C.c_int32, C.POINTER(C.c_float), C.c_int32],
    "epid_pf_bench_timed": [_P, _P, C.POINTER(PFParams), C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int32,
                            C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    "epid_starshot_analyze": [_P, _P, C.POINTER(StarParams), _P, _P, C.c_int32, _P],
    "epid_circle_profile": [_P, _P, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32, C.c_double, C.c_int32, C.c_double,
                            C.c_int32, C.c_int32, _P, _P, _P, C.POINTER(C.c_int32)],
    "epid_single_profile": [_P, _P, _P, C.c_int32, C.POINTER(SpParams), _P, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double,
                            C.c_double, C.c_double, _P, _P, _P, C.c_int32],
    "epid_field_profile_len": [C.c_int32, C.c_double, C.c_int32, C.c_double],
    "epid_field_analyze": [_P, _P, C.POINTER(FieldParams), _P, C.c_int32, _P, C.c_int32, _P],
    "epid_wl2d_analyze": [_P, _P, C.POINTER(WlParams), _P],
    "epid_zoom": [_P, _P, C.c_double, C.c_int32, C.c_int32, C.POINTER(_P)],
    "epid_rotate": [_P, _P, C.c_double, C.c_int32, C.POINTER(_P)],
    "epid_gamma": [_P, _P, _P, C.c_double, C.c_double, C.c_double, C.POINTER(_P)],
    "epid_gamma2d": [_P, _P, _P, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32, _P, _P, C.c_int32, C.c_int32,
                     C.POINTER(_P)],
    "epid_gamma_geometric": [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_double, C.c_double, _P, _P],
    "epid_gamma1d": [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, C.c_double, C.c_double, C.c_int32, C.c_double, _P, _P, _P],
    "epid_disk_locate": [_P, _P, _P, _P],
    "epid_roi_stats": [_P, _P, C.c_int32, _P, _P, _P, _P, _P, _P],
    "epid_weighted_centroid": [_P, _P, _P, _P, _P],
    "epid_disk_stats": [_P, _P, C.c_int32, _P, _P, _P, _P, _P, _P, _P],
    "epid_disk_percentiles": [_P, _P, C.c_int32, _P, C.c_int32, _P, _P],
    "epid_vmat_analyze": [_P, _P, _P, C.POINTER(VmatParams), _P],
    "epid_divide": [_P, _P, _P, _P, C.POINTER(_P)],
    "epid_dlg_analyze": [_P, _P, C.c_int32, _P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P],
    "epid_global_locate": [_P, _P, C.POINTER(LocateParams), _P, C.c_int32, _P, _P],
    "epid_lightrad_analyze": [_P, _P, C.POINTER(LrParams), _P],
    "epid_lightrad_stages": [_P, _P, C.POINTER(LrParams), _P, _P, _P, _P, _P],
    "epid_nm_uniformity": [_P, _P, C.c_int32, C.c_double, C.c_double, C.c_int32, C.c_double, _P, C.POINTER(_P), C.POINTER(_P)],
    "epid_nm_stages": [_P, _P, C.c_int32, C.c_double, C.c_double, C.c_int32, C.c_double, _P, _P, _P, _P, _P],
    "epid_nm_fov": [_P, _P, C.c_double, _P, C.POINTER(_P)],
    "epid_nt_slices": [_P, _P, C.c_int32, C.c_double, _P],
    "epid_nt_spheres": [_P, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P],
    "epid_tu_uniformity": [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_int32,
                           C.c_double, _P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P)],
    "epid_tu_stages": [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_int32, C.c_double,
                       _P, _P, _P, _P, _P, _P, _P],
    "epid_ct_localize": [_P, _P, _P, _P, _P, C.c_int32, C.c_double, C.c_int32, C.c_int32, C.c_double, _P, C.c_int32, _P, _P, _P, _P,
                         _P],
    "epid_ct_regions": [_P, _P, _P, _P, C.c_int32, C.c_double, _P, C.c_int32, _P, C.c_int32, _P, _P, _P],
    "epid_canny": [_P, _P, _P, C.c_int32, C.c_double, C.c_double, C.POINTER(_P)],
    "epid_hough_line": [_P, _P, C.c_int32, _P, C.POINTER(_P), C.POINTER(C.c_int32)],
    "epid_hough_candidates": [_P, _P, C.c_int32, C.c_int32, C.c_double, C.c_int32, _P, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                              C.POINTER(_P)],
    "epid_gather_i32": [_P, _P, C.c_int32, _P, _P],
    "epid_comm_unique_id": [_P],
    "epid_comm_init": [_P, C.c_int32, C.c_int32, _P],
    "epid_comm_destroy": [_P],
    "epid_comm_info": [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)],
    "epid_gather_results": [_P, _P, C.c_size_t, _P],
    "epid_barrier": [_P],
    "epid_xim_decode": [_P, _P, C.c_size_t, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, C.POINTER(_P)],
    "epid_log_fluence": [_P, _P, C.c_size_t, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_double, C.c_int32,
                         C.c_int32, C.c_int32, C.POINTER(_P), C.POINTER(_P)],
    "epid_hist_invert": [_P, _P, C.POINTER(_P), _P],
    "epid_gamma_stats": [_P, _P, _P, _P, _P],
    "epid_stack_mip": [_P, _P, C.POINTER(_P), C.POINTER(_P)],
    "epid_cbct_views": [_P, _P, _P, C.c_int32, C.POINTER(_P)],
}


def lib():
    """Load libepid.so (once).  Raises if the native extension has not been built."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise ImportError(
                        f"{LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(pylinac_b200 has no CPU fallback).")
                handle = C.CDLL(LIB_PATH)
                for name, args in _SIGNATURES.items():
                    fn = getattr(handle, name)
                    fn.argtypes = args
                    fn.restype = C.c_int32
                handle.epid_last_error.argtypes = []
                handle.epid_last_error.restype = C.c_char_p
                _lib = handle
    return _lib


def exported_symbols():
    return sorted(list(_SIGNATURES) + ["epid_last_error"])


def check(rc):
    if rc != EPID_OK:
        msg = lib().epid_last_error().decode("utf-8", "replace")
        if rc == ERR_NO_DEVICE:
            raise NoDeviceError(rc, msg)
        if rc == ERR_INVALID:
            raise ValueError(msg)
        raise NativeError(rc, msg)


def device_count() -> int:
    n = C.c_int32(0)
    check(lib().epid_device_count(C.byref(n)))
    return n.value


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Context:
    """One per device (epid_ctx)."""

    _default = {}

    def __init__(self, device: int = 0):
        h = _P()
        check(lib().epid_ctx_create(device, C.byref(h)))
        self.handle = h
        self.device = device

    @classmethod
    def default(cls, device: int | None = None) -> "Context":
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0")) if device_count() > 1 else 0
            if device >= device_count():
                device = 0
        if device not in cls._default:
            cls._default[device] = cls(device)
        return cls._default[device]

    def close(self):
        if self.handle:
            lib().epid_ctx_destroy(self.handle)
            self.handle = None

    def sync(self):
        check(lib().epid_sync(self.handle))

    def info(self):
        sm, ma, mi, mem = C.c_int32(), C.c_int32(), C.c_int32(), C.c_size_t()
        check(lib().epid_device_info(self.handle, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(mem)))
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "hbm_bytes": mem.value}

    def set_option(self, key: int, value: int) -> None:
        check(lib().epid_set_option(self.handle, key, value))

    def counter(self, key: int) -> int:
        v = C.c_int64()
        check(lib().epid_get_counter(self.handle, key, C.byref(v)))
        return v.value

    def comm_info(self) -> tuple[int, int]:
        """(nranks, rank) of this context's NCCL communicator; (1, 0) before parallel.init_comm."""
        n, r = C.c_int32(), C.c_int32()
        check(lib().epid_comm_info(self.handle, C.byref(n), C.byref(r)))
        return n.value, r.value

    def launches(self) -> int:
        n = C.c_int64()
        check(lib().epid_launch_count(self.handle, C.byref(n)))
        return n.value


class Batch:
    """n frames resident in HBM (epid_batch)."""

    def __init__(self, ctx: Context, handle):
        self.ctx = ctx
        self.handle = handle

    @classmethod
    def upload(cls, ctx: Context, arr: np.ndarray) -> "Batch":
        a = np.ascontiguousarray(arr)
        if a.ndim == 2:
            a = a[None]
        if a.ndim != 3:
            raise ValueError("expected [n, h, w] or [h, w]")
        if a.dtype not in _NP2DT:
            raise TypeError(f"unsupported dtype {a.dtype}")
        h = _P()
        check(lib().epid_batch_upload(ctx.handle, _ptr(a), _NP2DT[a.dtype], a.shape[0], a.shape[1], a.shape[2], C.byref(h)))
        return cls(ctx, h)

    @property
    def shape_dtype(self):
        dt, n, h, w = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        check(lib().epid_batch_shape(self.handle, C.byref(dt), C.byref(n), C.byref(h), C.byref(w)))
        return (n.value, h.value, w.value), _DT2NP[dt.value]

    def write(self, arr: np.ndarray) -> None:
        """overwrite the batch from a host array of the same shape / dtype (one H2D copy, synchronous)"""
        shape, dt = self.shape_dtype
        a = np.ascontiguousarray(arr)
        if a.shape != shape or a.dtype != dt:
            raise ValueError(f"expected {shape} {dt}, got {a.shape} {a.dtype}")
        check(lib().epid_batch_write(self.handle, _ptr(a)))

    def download(self) -> np.ndarray:
        shape, dt = self.shape_dtype
        out = np.empty(shape, dt)
        check(lib().epid_batch_download(self.handle, _ptr(out)))
        return out

    def free(self):
        if self.handle:
            lib().epid_batch_free(self.handle)
            self.handle = None

    def __enter__(self) -> "Batch":
        return self

    def __exit__(self, *exc) -> None:
        self.free()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def _unary2(self, fn, other: "Batch", *args) -> "Batch":
        h = _P()
        check(fn(self.ctx.handle, self.handle, other.handle, *args, C.byref(h)))
        return Batch(self.ctx, h)

    def _unary(self, fn, *args) -> "Batch":
        h = _P()
        check(fn(self.ctx.handle, self.handle, *args, C.byref(h)))
        return Batch(self.ctx, h)


@contextlib.contextmanager
def batch_for(ctx: Context, frames, dtype=None):
    """The Batch `frames`, or the ndarray `frames` ([n, h, w] or [h, w]) uploaded for the block and freed after it.  An ndarray
    that is not of `dtype` (when given) raises TypeError before anything reaches the device."""
    if isinstance(frames, Batch):
        yield frames
        return
    a = np.ascontiguousarray(frames)
    if a.ndim == 2:
        a = a[None]
    if dtype is not None and a.dtype != dtype:
        raise TypeError(f"{a.dtype} frames are not supported here; expected {np.dtype(dtype)}")
    with Batch.upload(ctx, a) as b:
        yield b


def pinned_empty(shape, dtype=np.uint16) -> np.ndarray:
    """numpy array backed by page-locked host memory (epid_host_alloc); freed when the array dies."""
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    p = _P()
    check(lib().epid_host_alloc(nbytes, C.byref(p)))
    import weakref

    buf = (C.c_char * max(nbytes, 1)).from_address(p.value)
    # every numpy view keeps `buf` alive through its .base chain; when the last one dies the block is unpinned and freed
    weakref.finalize(buf, _host_free, p.value)
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)


def _host_free(ptr: int) -> None:
    try:
        lib().epid_host_free(_P(ptr))
    except Exception:
        pass


class _PinnedPool:
    """Page-locked result buffers, recycled between calls.  cudaHostAlloc costs milliseconds and a fresh pageable
    ``np.zeros`` of a 30 MB result block costs thousands of first-touch page faults per call; a pooled pinned block costs
    neither and lets the library DMA the results straight into the array the caller receives.  A block returns to the pool
    when the last numpy view of it is garbage collected."""

    MAX_FREE_PER_SIZE = 4

    def __init__(self):
        self._free: dict[int, list[int]] = {}
        self._lock = threading.Lock()

    def take(self, shape, dtype) -> np.ndarray:
        import weakref

        dtype = np.dtype(dtype)
        nbytes = max(int(np.prod(shape)) * dtype.itemsize, 1)
        with self._lock:
            lst = self._free.get(nbytes)
            ptr = lst.pop() if lst else None
        if ptr is None:
            p = _P()
            check(lib().epid_host_alloc(nbytes, C.byref(p)))
            ptr = p.value
        buf = (C.c_char * nbytes).from_address(ptr)
        weakref.finalize(buf, self._give, nbytes, ptr)
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def _give(self, nbytes: int, ptr: int) -> None:
        with self._lock:
            lst = self._free.setdefault(nbytes, [])
            if len(lst) < self.MAX_FREE_PER_SIZE:
                lst.append(ptr)
                return
        try:
            lib().epid_host_free(_P(ptr))
        except Exception:
            pass


_RESULT_POOL = _PinnedPool()


XIM_OK, XIM_LOOKUP_CODE3, XIM_SHORT_BUFFER, XIM_U16_RANGE = 0, 1, 2, 3


def xim_decode(ctx: Context, arena: np.ndarray, desc: np.ndarray, h: int, w: int, bpp: int, dtype) -> tuple[Batch, np.ndarray]:
    """epid_xim_decode: arena (uint8, 16-byte aligned) + desc int64 [n, 4] -> (device Batch [n, h, w], int32 status [n])"""
    a = np.ascontiguousarray(arena, dtype=np.uint8)
    d = np.ascontiguousarray(desc, dtype=np.int64).reshape(-1, 4)
    if a.ctypes.data % 16:
        raise ValueError("the XIM arena must be 16-byte aligned")
    status = np.zeros(len(d), np.int32)
    h_out = _P()
    check(lib().epid_xim_decode(ctx.handle, _ptr(a), a.nbytes, _ptr(d), len(d), int(h), int(w), int(bpp), _NP2DT[np.dtype(dtype)],
                                _ptr(status), C.byref(h_out)))
    return Batch(ctx, h_out), status


LOG_DESC_DTYPE = np.dtype([("data_off", "<i8"), ("snap_stride", "<i8"), ("col_stride", "<i8"), ("f64", "<i4"), ("nsnap", "<i4"),
                           ("col_mu", "<i4", (2,)), ("col_x1", "<i4"), ("col_x2", "<i4"), ("col_leaf", "<i4", (2,)), ("num_pairs", "<i4"),
                           ("snap_off", "<i4"), ("nbeam", "<i4"), ("pair_off", "<i4"), ("row_off", "<i4"), ("flags", "<i4", (2,)),
                           ("pad", "<i4")])
assert LOG_DESC_DTYPE.itemsize == 88
LF_ZERO, LF_DIV25000 = 1, 2
PF_UNDER_JAW, PF_MOVED = 1, 2


def log_fluence(ctx: Context, arena: np.ndarray, logs: np.ndarray, snaps: np.ndarray, pair_flags: np.ndarray, rows: np.ndarray,
                resolution: float, w: int, h: int, kinds: int = 3) -> tuple[Batch | None, Batch | None]:
    """epid_log_fluence -> (actual, expected) float64 device batches [n, h, w] (None for a kind not requested)"""
    a = np.ascontiguousarray(arena).view(np.uint8).reshape(-1)
    d = np.ascontiguousarray(logs, dtype=LOG_DESC_DTYPE)
    s = np.ascontiguousarray(snaps, dtype=np.int32)
    pf = np.ascontiguousarray(pair_flags, dtype=np.uint8)
    r = np.ascontiguousarray(rows, dtype=np.int32)
    ha, he = _P(), _P()
    check(lib().epid_log_fluence(ctx.handle, _ptr(a), a.nbytes, _ptr(d), len(d), _ptr(s) if s.size else None, s.size, _ptr(pf), pf.size,
                                 _ptr(r), r.size, float(resolution), int(w), int(h), int(kinds), C.byref(ha), C.byref(he)))
    return (Batch(ctx, ha) if ha.value else None), (Batch(ctx, he) if he.value else None)


def hist_invert(ctx: Context, batch: Batch) -> tuple[Batch, np.ndarray]:
    """epid_hist_invert: check_inversion_by_histogram of every float64 frame -> (new batch, int32 inverted [n])"""
    (n, _, _), _ = batch.shape_dtype
    inv = np.zeros(n, np.int32)
    h = _P()
    check(lib().epid_hist_invert(ctx.handle, batch.handle, C.byref(h), _ptr(inv)))
    return Batch(ctx, h), inv


def gamma_stats(ctx: Context, gamma: Batch) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """epid_gamma_stats -> (sum of non-nan values, their count, count below 1) per frame"""
    (n, _, _), _ = gamma.shape_dtype
    s, c, p = np.zeros(n), np.zeros(n, np.int64), np.zeros(n, np.int64)
    check(lib().epid_gamma_stats(ctx.handle, gamma.handle, _ptr(s), _ptr(c), _ptr(p)))
    return s, c, p


def gamma2d(ctx: Context, ref: Batch, ev: Batch, dose_frac: float, threshold: float, cap: float, cap2: float, fill_value: float,
            global_dose: bool, offsets: np.ndarray, dist2: np.ndarray, full_search: bool = False) -> Batch:
    """epid_gamma2d -> float64 gamma maps [n, h, w] (device batch); offsets int32 [k, 2] and dist2 float64 [k] sorted by dist2"""
    o = np.ascontiguousarray(offsets, dtype=np.int32)
    d = np.ascontiguousarray(dist2, dtype=np.float64)
    h = _P()
    check(lib().epid_gamma2d(ctx.handle, ref.handle, ev.handle, float(dose_frac), float(threshold), float(cap), float(cap2),
                             float(fill_value), int(bool(global_dose)), _ptr(o), _ptr(d), len(d), int(bool(full_search)), C.byref(h)))
    return Batch(ctx, h)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def gamma_geometric(ctx: Context, eval_off, pt_off, decreasing, eval_x, eval_y, ref_x, ref_y, dta: float,
                    cap: float) -> tuple[np.ndarray, np.ndarray]:
    """epid_gamma_geometric -> (gamma float64 [points], svd_fail int32 [pairs]); packed host arrays, CSR offsets per pair"""
    eo, po, dec = _i64(eval_off), _i64(pt_off), np.ascontiguousarray(decreasing, dtype=np.int32)
    ex, ey, rx, ry = _f64(eval_x), _f64(eval_y), _f64(ref_x), _f64(ref_y)
    n = len(eo) - 1
    g, fail = np.empty(int(po[-1])), np.zeros(n, np.int32)
    check(lib().epid_gamma_geometric(ctx.handle, n, _ptr(eo), _ptr(po), _ptr(dec), _ptr(ex), _ptr(ey), _ptr(rx), _ptr(ry), float(dta),
                                     float(cap), _ptr(g), _ptr(fail)))
    return g, fail


def gamma1d(ctx: Context, eval_off, pt_off, dose_f32, eval_x, eval_y, ref_x, ref_y, dose_ta2, dta: float, dta2: float, num: int,
            cap: float) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """epid_gamma1d -> (gamma [points], samples [points, num], sample x [points, num]), float64; packed host arrays, CSR offsets"""
    eo, po, f32 = _i64(eval_off), _i64(pt_off), np.ascontiguousarray(dose_f32, dtype=np.int32)
    ex, ey, rx, ry, d2 = _f64(eval_x), _f64(eval_y), _f64(ref_x), _f64(ref_y), _f64(dose_ta2)
    n, k = len(eo) - 1, int(po[-1])
    g, s, x = np.empty(k), np.empty((k, num)), np.empty((k, num))
    check(lib().epid_gamma1d(ctx.handle, n, _ptr(eo), _ptr(po), _ptr(f32), _ptr(ex), _ptr(ey), _ptr(rx), _ptr(ry), _ptr(d2), float(dta),
                             float(dta2), int(num), float(cap), _ptr(g), _ptr(s), _ptr(x)))
    return g, s, x


def _unsupported_as_not_implemented(rc):
    try:
        check(rc)
    except NativeError as e:
        if e.code == ERR_UNSUPPORTED:
            raise NotImplementedError(e.msg) from None
        raise


def stack_mip(ctx: Context, volume: Batch) -> tuple[Batch, Batch]:
    """epid_stack_mip: volume [N, H, W] int16 / uint16 -> (colmax [W, 1, N], rowmax [H, 1, N]) device batches of the volume's dtype:
    np.stack(slices, axis=-1).max(axis=0) / .max(axis=1).  Other dtypes raise NotImplementedError."""
    hc, hr = _P(), _P()
    _unsupported_as_not_implemented(lib().epid_stack_mip(ctx.handle, volume.handle, C.byref(hc), C.byref(hr)))
    return Batch(ctx, hc), Batch(ctx, hr)


def cbct_views(ctx: Context, z0: Batch, z1: Batch | None, src_dtype) -> Batch:
    """epid_cbct_views: zoomed projections (float64 [P, 1, N']) -> uint16 frames [2 or 4, N', P]: rot90 and fliplr(rot90) of z0, then
    of z1, rounded like scipy's integer zoom output of `src_dtype` and stored as the uint16 bits of that dtype."""
    h = _P()
    _unsupported_as_not_implemented(lib().epid_cbct_views(ctx.handle, z0.handle, None if z1 is None else z1.handle,
                                                          _NP2DT[np.dtype(src_dtype)], C.byref(h)))
    return Batch(ctx, h)


def frame_stats(ctx: Context, batch: Batch, view=None, percentiles=()):
    (n, h, w), _ = batch.shape_dtype
    r0, c0, vh, vw = view if view is not None else (0, 0, h, w)
    q = np.asarray(percentiles, dtype=np.float64)
    nq = q.size
    mn, mx, sm = np.empty(n), np.empty(n), np.empty(n)
    rows, cols = np.empty((n, vh)), np.empty((n, vw))
    pct = np.empty((n, max(nq, 1)))
    check(lib().epid_frame_stats(ctx.handle, batch.handle, r0, c0, vh, vw, _ptr(q) if nq else None, nq, _ptr(mn), _ptr(mx),
                                 _ptr(sm), _ptr(rows), _ptr(cols), _ptr(pct)))
    return {"min": mn, "max": mx, "sum": sm, "rowsum": rows, "colsum": cols, "percentiles": pct[:, :nq]}


def frame_histogram(ctx: Context, batch: Batch, view=None) -> np.ndarray:
    (n, h, w), _ = batch.shape_dtype
    r0, c0, vh, vw = view if view is not None else (0, 0, h, w)
    hist = np.empty((n, 65536), np.uint32)
    check(lib().epid_frame_histogram(ctx.handle, batch.handle, r0, c0, vh, vw, _ptr(hist)))
    return hist


def find_peaks(ctx: Context, values, threshold=-np.inf, peak_separation=0, max_number=None, fwxm_height=0.5, min_width=0,
               search_region=(0.0, 1.0), peak_sort="prominences", required_prominence=None):
    v = np.ascontiguousarray(values, dtype=np.float64)
    n = v.size
    p = PeakParams(float(threshold), float(peak_separation), PEAKS_ALL if max_number is None else int(max_number), float(fwxm_height),
                   float(min_width), float(search_region[0]), float(search_region[1]), 1 if peak_sort == "peak_heights" else 0,
                   -1.0 if required_prominence is None else float(required_prominence))
    cap = n // 2 + 2
    idx = np.empty(cap, np.int64)
    lb, rb = np.empty(cap, np.int64), np.empty(cap, np.int64)
    hts, prom, wid, wh, lip, rip = (np.empty(cap) for _ in range(6))
    cnt = C.c_int32()
    check(lib().epid_find_peaks(ctx.handle, _ptr(v), n, C.byref(p), cap, _ptr(idx), _ptr(hts), _ptr(prom), _ptr(lb), _ptr(rb),
                                _ptr(wid), _ptr(wh), _ptr(lip), _ptr(rip), C.byref(cnt)))
    c = cnt.value
    props = {"peak_heights": hts[:c].copy(), "prominences": prom[:c].copy(), "left_bases": lb[:c].copy(),
             "right_bases": rb[:c].copy(), "widths": wid[:c].copy(), "width_heights": wh[:c].copy(),
             "left_ips": lip[:c].copy(), "right_ips": rip[:c].copy()}
    return idx[:c].copy(), props


def pf_analyze(ctx: Context, frames, params: PFParams, meas_cap: int = 1024, host_pipeline: bool = False):
    """frames: a Batch (device-resident) or a uint16 ndarray [n,h,w] (host; chunked H2D overlapped with compute)."""
    if isinstance(frames, Batch):
        (n, _, _), _ = frames.shape_dtype
        summ = np.zeros(n, PF_SUMMARY_DTYPE)
        meas = np.zeros((n, meas_cap), PF_MEAS_DTYPE)
        check(lib().epid_pf_analyze(ctx.handle, frames.handle, C.byref(params), _ptr(summ), _ptr(meas), meas_cap))
        return summ, meas
    a = frames
    if a.dtype != np.uint16:
        raise TypeError("picket fence frames must be uint16")
    if a.ndim == 2:
        a = a[None]
    a = np.ascontiguousarray(a)
    n, h, w = a.shape
    # every element of both blocks is overwritten by the device-to-host copy of the (zero-initialised) device result arrays
    summ = _RESULT_POOL.take((n,), PF_SUMMARY_DTYPE)
    meas = _RESULT_POOL.take((n, meas_cap), PF_MEAS_DTYPE)
    check(lib().epid_pf_analyze_host(ctx.handle, _ptr(a), n, h, w, C.byref(params), _ptr(summ), _ptr(meas), meas_cap))
    return summ, meas


def pf_bench(ctx: Context, batch: Batch, params: PFParams, iters: int):
    total, stats = C.c_float(), C.c_float()
    launches = C.c_int64()
    check(lib().epid_pf_bench(ctx.handle, batch.handle, C.byref(params), iters, C.byref(total), C.byref(stats), C.byref(launches)))
    return total.value, stats.value, launches.value


PF_STAGE_NAMES = ("k_pf_init + k_pf_pilot", "k_pf_stream", "k_pf_tail", "k_pf_windows_fast", "k_pf_windows (generic)", "k_pf_finalize",
                  "exact front end (fallback)", "k_pf_win_medians", "k_pf_win_fwxm")


def pf_bench_timed(ctx: Context, batch: Batch, params: PFParams, iters: int):
    """(total_ms of `iters` passes, {stage name: ms per pass}, launches, frames re-run by the per-frame fallback)"""
    out = (C.c_float * 16)()
    total = C.c_float()
    launches, redone = C.c_int64(), C.c_int64()
    check(lib().epid_pf_bench_timed(ctx.handle, batch.handle, C.byref(params), iters, C.byref(total), out, 16, C.byref(launches),
                                    C.byref(redone)))
    return total.value, {name: out[k] / iters for k, name in enumerate(PF_STAGE_NAMES)}, launches.value, redone.value


def pf_bench_stages(ctx: Context, batch: Batch, params: PFParams, iters: int) -> dict:
    """{stage name: ms per pass} from CUDA events recorded between the kernels of `iters` device-resident passes."""
    out = (C.c_float * 16)()
    check(lib().epid_pf_bench_stages(ctx.handle, batch.handle, C.byref(params), iters, out, 16))
    return {name: out[k] / iters for k, name in enumerate(PF_STAGE_NAMES)}


def gaussian_kernel_table(max_sigma: int):
    """scipy/ndimage/_filters.py:_gaussian_kernel1d (order 0, truncate 4) for sigma = 1 .. max_sigma, concatenated.
    Host-side table of filter weights (the same numpy expression scipy evaluates); offsets[s] = start of sigma s."""
    offsets = np.zeros(max_sigma + 1, np.int32)
    chunks = []
    pos = 0
    for s in range(1, max_sigma + 1):
        sd = float(s)
        lw = int(4.0 * sd + 0.5)
        x = np.arange(-lw, lw + 1)
        phi = np.exp(-0.5 / (sd * sd) * x**2)
        w = (phi / phi.sum())[::-1]
        offsets[s] = pos
        chunks.append(np.ascontiguousarray(w, dtype=np.float64))
        pos += w.size
    return np.concatenate(chunks), offsets


def starshot_analyze(ctx: Context, frames, params: StarParams) -> np.ndarray:
    """frames: a Batch (device-resident, uint16) or a uint16 ndarray [n,h,w] / [h,w]; one STAR_RESULT_DTYPE row per frame."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, h, w), _ = b.shape_dtype
        # CollapsedCircleProfile length <= 2 pi * 1.1 * 0.95 * (dim / 2) * 3; sigma = round(0.003 * length)
        max_sigma = max(int(round(0.003 * (10 * max(h, w) + 64))) + 1, 2)
        gw, go = gaussian_kernel_table(max_sigma)
        res = np.zeros(n, STAR_RESULT_DTYPE)
        check(lib().epid_starshot_analyze(ctx.handle, b.handle, C.byref(params), _ptr(gw), _ptr(go), max_sigma, _ptr(res)))
    return res


def gaussian_kernel1d(sigma: float, truncate: float = 4.0):
    """scipy/ndimage/_filters.py:_gaussian_kernel1d (order 0), reversed as gaussian_filter1d hands it to correlate1d."""
    sd = float(sigma)
    lw = int(truncate * sd + 0.5)
    x = np.arange(-lw, lw + 1)
    phi = np.exp(-0.5 / (sd * sd) * x**2)
    return np.ascontiguousarray((phi / phi.sum())[::-1], dtype=np.float64), lw


def field_analyze(ctx: Context, frames, params: FieldParams) -> np.ndarray:
    """frames: a Batch (device-resident, uint16) or a uint16 ndarray [n,h,w] / [h,w]; one FIELD_RESULT_DTYPE row per frame."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, h, w), _ = b.shape_dtype
        gh = gv = None
        lh = lv = 0
        if params.edge != 0:
            # gaussian_filter1d(values, sigma=edge_smoothing_ratio * len(values)) (core/profile.py:1655-1659): one table per profile length
            nh = lib().epid_field_profile_len(w, params.dpmm, params.interpolation, params.interpolation_resolution_mm)
            nv = lib().epid_field_profile_len(h, params.dpmm, params.interpolation, params.interpolation_resolution_mm)
            gh, lh = gaussian_kernel1d(params.edge_smoothing_ratio * nh)
            gv, lv = gaussian_kernel1d(params.edge_smoothing_ratio * nv)
        res = np.zeros(n, FIELD_RESULT_DTYPE)
        check(lib().epid_field_analyze(ctx.handle, b.handle, C.byref(params), _ptr(gh), lh, _ptr(gv), lv, _ptr(res)))
    return res


def wl2d_analyze(ctx: Context, frames, params: WlParams) -> np.ndarray:
    """frames: a Batch (device-resident, uint16) or a uint16 ndarray [n,h,w] / [h,w]; one WL_RESULT_DTYPE row per frame."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        res = np.zeros(n, WL_RESULT_DTYPE)
        check(lib().epid_wl2d_analyze(ctx.handle, b.handle, C.byref(params), _ptr(res)))
    return res


def disk_locate(ctx: Context, frames, params: DiskParams) -> np.ndarray:
    """SizedDiskRegion / SizedDiskLocator on uint16 frames: one DISK_RESULT_DTYPE row per frame."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        res = np.zeros(n, DISK_RESULT_DTYPE)
        check(lib().epid_disk_locate(ctx.handle, b.handle, C.byref(params), _ptr(res)))
    return res


def roi_stats(ctx: Context, frames, verts_xy) -> dict:
    """RectangleROI statistics: verts_xy [nroi, 4, 2] corner (x, y) -> dict of [n, nroi] arrays (count, mean, std, min, max)."""
    v = np.ascontiguousarray(verts_xy, dtype=np.float64).reshape(-1, 4, 2)
    with batch_for(ctx, frames) as b:
        (n, _, _), _ = b.shape_dtype
        out = {k: np.empty((n, len(v))) for k in ("count", "mean", "std", "min", "max")}
        check(lib().epid_roi_stats(ctx.handle, b.handle, len(v), _ptr(v), _ptr(out["count"]), _ptr(out["mean"]), _ptr(out["std"]),
                                   _ptr(out["min"]), _ptr(out["max"])))
    return out


DISK_STATS = ("count", "mean", "std", "min", "max", "median")


def disk_stats(ctx: Context, frames, disks) -> dict:
    """DiskROI statistics of a batch: disks [ndisk, 4] rows (frame index, centre row, centre column, radius) -> dict of [ndisk]
    float64 arrays (count, mean, std, min, max, median), each numpy's value over arr[skimage.draw.disk((cy, cx), r)] of that frame."""
    d = np.ascontiguousarray(disks, dtype=np.float64).reshape(-1, 4)
    out = {k: np.empty(len(d)) for k in DISK_STATS}
    with batch_for(ctx, frames) as b:
        check(lib().epid_disk_stats(ctx.handle, b.handle, len(d), _ptr(d), *(_ptr(out[k]) for k in DISK_STATS)))
    return out


def disk_percentiles(ctx: Context, frames, disks, q) -> np.ndarray:
    """np.percentile(arr[skimage.draw.disk((cy, cx), r)], q) of each disk of `disks` (rows as for disk_stats) for each q of `q` (1 to 16
    Python numbers) -> float64 [ndisk, nq].  A float32 batch gives numpy's float32 values.  NaN for a disk with a NaN pixel or no pixel."""
    d = np.ascontiguousarray(disks, dtype=np.float64).reshape(-1, 4)
    qs = np.ascontiguousarray(q, dtype=np.float64).reshape(-1)
    out = np.empty((len(d), len(qs)))
    with batch_for(ctx, frames) as b:
        check(lib().epid_disk_percentiles(ctx.handle, b.handle, len(d), _ptr(d), len(qs), _ptr(qs), _ptr(out)))
    return out


def vmat_analyze(ctx: Context, img1, img2, params: VmatParams) -> np.ndarray:
    """n (image 1, image 2) pairs of uint16 frames (Batch or ndarray [n,h,w] / [h,w]) -> one VMAT_RESULT_DTYPE row per pair."""
    with batch_for(ctx, img1, np.uint16) as b1, batch_for(ctx, img2, np.uint16) as b2:
        (n, _, _), _ = b1.shape_dtype
        res = np.zeros(n, VMAT_RESULT_DTYPE)
        check(lib().epid_vmat_analyze(ctx.handle, b1.handle, b2.handle, C.byref(params), _ptr(res)))
    return res


def lightrad_analyze(ctx: Context, frames, params: LrParams) -> np.ndarray:
    """Light / radiation field coincidence on uint16 frames (Batch or ndarray [n,h,w] / [h,w]) -> one LR_RESULT_DTYPE row per frame."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        res = np.zeros(n, LR_RESULT_DTYPE)
        check(lib().epid_lightrad_analyze(ctx.handle, b.handle, C.byref(params), _ptr(res)))
    return res


LR_INFO_FIELDS = ("mn", "mx", "sum", "corner", "checked", "inv", "near_mask", "fmn", "fmx", "umin", "umax")


def lightrad_stages(ctx: Context, frames, params: LrParams) -> dict:
    """Diagnostic read-back of epid_lightrad_stages: {"results": LR_RESULT_DTYPE rows, "filtered", "equalised", "equalised_filtered":
    uint16 [n, h, w], "info": {name: int64 [n]} for the names of LR_INFO_FIELDS}.  The equalised planes and fmn .. umax of frames
    without a near-edge BB are unspecified."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, h, w), _ = b.shape_dtype
        res = np.zeros(n, LR_RESULT_DTYPE)
        planes = [np.empty((n, h, w), np.uint16) for _ in range(3)]
        info = np.zeros((n, len(LR_INFO_FIELDS)), np.int64)
        check(lib().epid_lightrad_stages(ctx.handle, b.handle, C.byref(params), _ptr(res), *[_ptr(a) for a in planes], _ptr(info)))
    return {"results": res, "filtered": planes[0], "equalised": planes[1], "equalised_filtered": planes[2],
            "info": {name: info[:, k] for k, name in enumerate(LR_INFO_FIELDS)}}


def nm_uniformity(ctx: Context, frames, bin_size: int, ufov_erode: float, cfov_erode: float, window: int, threshold: float,
                  arrays: bool = True):
    """epid_nm_uniformity on uint16 frames (Batch or ndarray [n,h,w] / [h,w]) -> (NM_RESULT_DTYPE rows, cleaned, masks): cleaned is a
    float64 device Batch [n, hb, wb] and masks a uint8 device Batch [2n, hb, wb] (UFOV, CFOV of each frame), both None when not
    `arrays`.  Unsupported dtypes and bin sizes raise NotImplementedError."""
    with batch_for(ctx, frames) as b:
        (n, _, _), _ = b.shape_dtype
        res = np.zeros(n, NM_RESULT_DTYPE)
        hc, hm = _P(), _P()
        _unsupported_as_not_implemented(lib().epid_nm_uniformity(
            ctx.handle, b.handle, int(bin_size), float(ufov_erode), float(cfov_erode), int(window), float(threshold), _ptr(res),
            C.byref(hc) if arrays else None, C.byref(hm) if arrays else None))
    if not arrays:
        return res, None, None
    return res, Batch(ctx, hc), Batch(ctx, hm)


def nm_stages(ctx: Context, frames, bin_size: int, ufov_erode: float, cfov_erode: float, window: int, threshold: float) -> dict:
    """Diagnostic read-back of epid_nm_stages: {"results", "filtered" (uint32 S after the filter), "cleaned" (uint32 S after the
    threshold and the stray-pixel stencil), "edt2" (int32 squared EDT, -1 for a frame without a component), "masks" (uint8
    [n, 2, hb, wb])}."""
    with batch_for(ctx, frames) as b:
        (n, h, w), _ = b.shape_dtype
        hb, wb = -(-h // int(bin_size)), -(-w // int(bin_size))
        res = np.zeros(n, NM_RESULT_DTYPE)
        filt, clean = np.empty((n, hb, wb), np.uint32), np.empty((n, hb, wb), np.uint32)
        edt2, masks = np.empty((n, hb, wb), np.int32), np.empty((n, 2, hb, wb), np.uint8)
        _unsupported_as_not_implemented(lib().epid_nm_stages(
            ctx.handle, b.handle, int(bin_size), float(ufov_erode), float(cfov_erode), int(window), float(threshold), _ptr(res),
            _ptr(filt), _ptr(clean), _ptr(edt2), _ptr(masks)))
    return {"results": res, "filtered": filt, "cleaned": clean, "edt2": edt2, "masks": masks}


def nm_fov(ctx: Context, binary: np.ndarray, erode: float) -> tuple[np.ndarray, np.ndarray]:
    """epid_nm_fov on one 2-D binary frame -> (NM_RESULT_DTYPE row, eroded uint8 mask)"""
    a = np.ascontiguousarray(binary, dtype=np.uint8)[None]
    res = np.zeros(1, NM_RESULT_DTYPE)
    with Batch.upload(ctx, a) as b:
        h = _P()
        check(lib().epid_nm_fov(ctx.handle, b.handle, float(erode), _ptr(res), C.byref(h)))
        with Batch(ctx, h) as m:
            mask = m.download()[0]
    return res[0], mask


def nt_slices(ctx: Context, volumes, nz: int, ufov_erode: float) -> np.ndarray:
    """epid_nt_slices on uint16 volumes (Batch of n x nz slices, or ndarray [n, nz, h, w]) -> one NT_SLICE_DTYPE row per slice,
    [n * nz]"""
    with batch_for(ctx, _volume_batch(volumes), np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        res = np.zeros(n, NT_SLICE_DTYPE)
        _unsupported_as_not_implemented(lib().epid_nt_slices(ctx.handle, b.handle, int(nz), float(ufov_erode), _ptr(res)))
    return res


def nt_spheres(ctx: Context, volumes, nz: int, spheres: np.ndarray, maxfun: int = 600, maxiter: int = 600) -> np.ndarray:
    """epid_nt_spheres: the sphere searches of `spheres` (NT_SPHERE_IN_DTYPE rows) in uint16 volumes (Batch of n x nz slices, or
    ndarray [n, nz, h, w]) -> one NT_SPHERE_DTYPE row per sphere"""
    spheres = np.ascontiguousarray(spheres, NT_SPHERE_IN_DTYPE)
    with batch_for(ctx, _volume_batch(volumes), np.uint16) as b:
        res = np.zeros(len(spheres), NT_SPHERE_DTYPE)
        _unsupported_as_not_implemented(lib().epid_nt_spheres(ctx.handle, b.handle, int(nz), _ptr(spheres), len(spheres), int(maxfun),
                                                              int(maxiter), _ptr(res)))
    return res


def _volume_batch(volumes):
    """[n, nz, h, w] ndarray volumes as n x nz slices; a Batch as is"""
    if isinstance(volumes, Batch):
        return volumes
    return np.ascontiguousarray(volumes).reshape(-1, *np.shape(volumes)[-2:])


def tu_uniformity(ctx: Context, volumes, nz: int, first: int, count: int, bin_size: int, erode, window: int, threshold: float,
                  arrays: bool = True):
    """epid_tu_uniformity on uint16 volumes (Batch of n x nz slices, or ndarray [n, nz, h, w]) with the slab [first, first + count) and
    erode = (UFOV, CFOV, center) 1 - size -> (TU_RESULT_DTYPE rows, mean, cleaned, masks): device Batches of the float64 slab means
    [n, h, w], the float64 cleaned frames [n, hb, wb] and the uint8 masks [3n, hb, wb], all None when not `arrays`."""
    with batch_for(ctx, _volume_batch(volumes), np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        res = np.zeros(n // int(nz), TU_RESULT_DTYPE)
        hs = [_P(), _P(), _P()]
        _unsupported_as_not_implemented(lib().epid_tu_uniformity(
            ctx.handle, b.handle, int(nz), int(first), int(count), int(bin_size), *(float(e) for e in erode), int(window),
            float(threshold), _ptr(res), *(C.byref(h) if arrays else None for h in hs)))
    if not arrays:
        return res, None, None, None
    return (res, *(Batch(ctx, h) for h in hs))


def tu_stages(ctx: Context, volumes, nz: int, first: int, count: int, bin_size: int, erode, window: int, threshold: float) -> dict:
    """Diagnostic read-back of epid_tu_stages: {"results", "mean" [n, h, w], "binned", "filtered", "cleaned" (float64 [n, hb, wb]),
    "edt2" (int32 squared EDT, -1 for a volume without a component), "masks" (uint8 [n, 3, hb, wb])}."""
    with batch_for(ctx, _volume_batch(volumes), np.uint16) as b:
        (n, h, w), _ = b.shape_dtype
        nv = n // int(nz)
        hb, wb = -(-h // int(bin_size)), -(-w // int(bin_size))
        res = np.zeros(nv, TU_RESULT_DTYPE)
        out = {"mean": np.empty((nv, h, w)), "binned": np.empty((nv, hb, wb)), "filtered": np.empty((nv, hb, wb)),
               "cleaned": np.empty((nv, hb, wb)), "edt2": np.empty((nv, hb, wb), np.int32), "masks": np.empty((nv, 3, hb, wb), np.uint8)}
        _unsupported_as_not_implemented(lib().epid_tu_stages(
            ctx.handle, b.handle, int(nz), int(first), int(count), int(bin_size), *(float(e) for e in erode), int(window),
            float(threshold), _ptr(res), *(_ptr(a) for a in out.values())))
    out["results"] = res
    return out


def ct_localize(ctx: Context, volume, slope, intercept, slices, catphan_size: float, clear_borders: bool,
                clip_in_localization: bool = True, stages: bool = False, otsu_disk_radius: float = 0.0):
    """epid_ct_localize: the phantom localization of `slices` of an int16 / uint16 series (Batch [n, h, w] or ndarray) with per-slice
    slope / intercept [n] -> CT_SLICE_DTYPE rows [len(slices)]; with `stages`, (rows, {"scharr", "smoothed" (float64), "filled" (bool),
    "labels" (int32 skimage labels, 0 off the mask)} planes [len(slices), h, w]).  otsu_disk_radius > 0 (pixels) with
    clip_in_localization False is get_regions' Slice branch; 0 with clip_in_localization True its ndarray branch."""
    sl = np.ascontiguousarray(slices, dtype=np.int32).reshape(-1)
    w, lw = gaussian_kernel1d(1.0)
    with batch_for(ctx, volume) as b:
        (n, h, wd), _ = b.shape_dtype
        sp = np.ascontiguousarray(np.broadcast_to(np.asarray(slope, np.float64), (n,)))
        ic = np.ascontiguousarray(np.broadcast_to(np.asarray(intercept, np.float64), (n,)))
        res = np.zeros(len(sl), CT_SLICE_DTYPE)
        planes = None
        if stages:
            m = len(sl)
            planes = {"scharr": np.empty((m, h, wd)), "smoothed": np.empty((m, h, wd)), "filled": np.empty((m, h, wd), np.uint8),
                      "labels": np.empty((m, h, wd), np.int32)}
        _unsupported_as_not_implemented(lib().epid_ct_localize(
            ctx.handle, b.handle, _ptr(sp), _ptr(ic), _ptr(sl), len(sl), float(catphan_size), int(bool(clear_borders)),
            int(bool(clip_in_localization)), float(otsu_disk_radius), _ptr(w), int(lw), _ptr(res), *(_ptr(a) for a in (planes or {}).values()),
            *((None,) * (0 if planes else 4))))
    if not stages:
        return res
    planes["filled"] = planes["filled"].view(bool)
    lab = planes["labels"].reshape(len(sl), -1)
    for k in range(len(sl)):      # union-find roots (indices within the slice) -> labels 1.. in raster order of each region's first pixel
        fg = lab[k] >= 0
        _, inv = np.unique(lab[k][fg], return_inverse=True)
        out = np.zeros(lab.shape[1], np.int32)
        out[fg] = inv + 1
        lab[k] = out
    return res, planes


def ct_regions(ctx: Context, volume, slope, intercept, slice_num: int, otsu_disk_radius: float, capacity: int = 64):
    """epid_ct_regions: get_regions(slice) of slice `slice_num` of an int16 / uint16 series (Batch [n, h, w] or ndarray) with per-slice
    slope / intercept [n] -> (CT_REGION_DTYPE rows in label order, threshold, max_edge).  A table longer than `capacity` is read again
    with room for all of it."""
    w, lw = gaussian_kernel1d(1.0)
    with batch_for(ctx, volume) as b:
        (n, _, _), _ = b.shape_dtype
        sp = np.ascontiguousarray(np.broadcast_to(np.asarray(slope, np.float64), (n,)))
        ic = np.ascontiguousarray(np.broadcast_to(np.asarray(intercept, np.float64), (n,)))
        cap = max(int(capacity), 1)
        while True:
            rows = np.zeros(cap, CT_REGION_DTYPE)
            count, thres, max_edge = C.c_int32(), C.c_double(), C.c_double()
            _unsupported_as_not_implemented(lib().epid_ct_regions(
                ctx.handle, b.handle, _ptr(sp), _ptr(ic), int(slice_num), float(otsu_disk_radius), _ptr(w), int(lw), _ptr(rows), cap,
                C.byref(count), C.byref(thres), C.byref(max_edge)))
            if count.value <= cap:
                return rows[:count.value], thres.value, max_edge.value
            cap = count.value


def divide(ctx: Context, num, den, sign_off=None) -> np.ndarray:
    """num / den as float64 (uint16 or float64 inputs of equal shape); sign_off [n, 2, 2] = (sign, offset) of num / den per frame."""
    a, b = np.ascontiguousarray(num), np.ascontiguousarray(den)
    squeeze = a.ndim == 2
    if a.dtype != b.dtype or a.dtype not in (np.uint16, np.float64):
        a, b = a.astype(np.float64), b.astype(np.float64)
    so = None if sign_off is None else np.ascontiguousarray(sign_off, dtype=np.float64).reshape(-1, 4)
    h = _P()
    with Batch.upload(ctx, a) as ba, Batch.upload(ctx, b) as bb:
        check(lib().epid_divide(ctx.handle, ba.handle, bb.handle, _ptr(so), C.byref(h)))
        with Batch(ctx, h) as out:
            r = out.download()
    return r[0] if squeeze else r


def dlg_analyze(ctx: Context, frames, bottom, top, c0: int, c1: int, planned):
    """-> (measured [n, nleaf], slope [n], intercept [n], dlg [n]) for uint16 frames."""
    bot = np.ascontiguousarray(bottom, dtype=np.int32)
    tp = np.ascontiguousarray(top, dtype=np.int32)
    pl = np.ascontiguousarray(planned, dtype=np.float64)
    nleaf = len(bot)
    with batch_for(ctx, frames, np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        meas, slope, icpt, dlg = np.empty((n, nleaf)), np.empty(n), np.empty(n), np.empty(n)
        check(lib().epid_dlg_analyze(ctx.handle, b.handle, nleaf, _ptr(bot), _ptr(tp), int(c0), int(c1), _ptr(pl), _ptr(meas), _ptr(slope),
                                     _ptr(icpt), _ptr(dlg)))
    return meas, slope, icpt, dlg


def global_locate(ctx: Context, frames, params: LocateParams, region_cap: int = 1024):
    """Whole-frame threshold sweep: -> list (per frame) of REGION_DTYPE arrays in the reference's visiting order."""
    with batch_for(ctx, frames, np.uint16) as b:
        (n, _, _), _ = b.shape_dtype
        regs = np.zeros((n, region_cap), REGION_DTYPE)
        counts, flags = np.zeros(n, np.int32), np.zeros(n, np.int32)
        check(lib().epid_global_locate(ctx.handle, b.handle, C.byref(params), _ptr(regs), int(region_cap), _ptr(counts), _ptr(flags)))
    if (flags != 0).any():
        raise MemoryError(f"global locator: device lists overflowed (flags {flags.tolist()}); raise region_cap or pre-filter the frame")
    return [regs[i, : counts[i]].copy() for i in range(n)]


def canny(ctx: Context, image: np.ndarray, sigma: float = 1.0, low_threshold: float = 0.1, high_threshold: float = 0.2) -> np.ndarray:
    """skimage.feature.canny semantics for a float64 image [h, w] (or [n, h, w]) -> boolean edge map(s)."""
    a = np.ascontiguousarray(image, dtype=np.float64)
    squeeze = a.ndim == 2
    w, lw = gaussian_kernel1d(float(sigma))
    h = _P()
    with Batch.upload(ctx, a) as b:
        check(lib().epid_canny(ctx.handle, b.handle, _ptr(w), int(lw), float(low_threshold), float(high_threshold), C.byref(h)))
        with Batch(ctx, h) as out:
            r = out.download()
    r = r.astype(bool)
    return r[0] if squeeze else r


def hough_line(ctx: Context, edges: np.ndarray, theta: np.ndarray):
    """skimage.transform.hough_line: -> (accumulator Batch [1, 2 * offset + 1, ntheta] int32 on the device, offset)"""
    e = np.ascontiguousarray(edges).astype(np.uint8)
    th = np.ascontiguousarray(theta, dtype=np.float64)
    h, off = _P(), C.c_int32()
    with Batch.upload(ctx, e) as b:
        check(lib().epid_hough_line(ctx.handle, b.handle, len(th), _ptr(th), C.byref(h), C.byref(off)))
    return Batch(ctx, h), off.value


def hough_candidates(ctx: Context, accum: Batch, min_xdistance: int, min_ydistance: int, threshold: float | None = None, cap: int = 1 << 16):
    """-> (candidates [k, 3] (row, col, value), global maximum, max-filtered accumulator Batch)"""
    cand = np.zeros((cap, 3), np.int32)
    cnt, gmax = C.c_int32(), C.c_int32()
    h = _P()
    check(lib().epid_hough_candidates(ctx.handle, accum.handle, int(min_xdistance), int(min_ydistance), -1.0 if threshold is None else float(threshold),
                                      cap, _ptr(cand), C.byref(cnt), C.byref(gmax), C.byref(h)))
    return cand[: cnt.value].copy(), gmax.value, Batch(ctx, h)


def gather_i32(ctx: Context, img: Batch, yx: np.ndarray) -> np.ndarray:
    pts = np.ascontiguousarray(yx, dtype=np.int32).reshape(-1, 2)
    out = np.zeros(len(pts), np.int32)
    check(lib().epid_gather_i32(ctx.handle, img.handle, len(pts), _ptr(pts), _ptr(out)))
    return out


def weighted_centroid(ctx: Context, frames):
    """(cx, cy, total) arrays of length n: sum(x * a) / sum(a), sum(y * a) / sum(a), sum(a)."""
    with batch_for(ctx, frames) as b:
        (n, _, _), _ = b.shape_dtype
        cx, cy, tot = np.empty(n), np.empty(n), np.empty(n)
        check(lib().epid_weighted_centroid(ctx.handle, b.handle, _ptr(cx), _ptr(cy), _ptr(tot)))
    return cx, cy, tot


def circle_profile(ctx: Context, image: np.ndarray, center, radius: float, start_angle: float = 0.0, ccw: bool = True,
                   sampling_ratio: float = 1.0, collapsed: bool = False, width_ratio: float = 0.1, num_profiles: int = 20):
    """(profile, x_locations, y_locations) of a CircleProfile / CollapsedCircleProfile of one image."""
    a = np.ascontiguousarray(image)
    if a.dtype not in (np.uint8, np.uint16, np.float32, np.float64):
        a = a.astype(np.float64)
    rmax = radius * (1 + width_ratio) if collapsed else radius
    cap = int(np.ceil(2 * np.pi * rmax * sampling_ratio)) + 8
    prof, xl, yl = np.empty(cap), np.empty(cap), np.empty(cap)
    cnt = C.c_int32()
    with Batch.upload(ctx, a) as b:
        check(lib().epid_circle_profile(ctx.handle, b.handle, float(center[0]), float(center[1]), float(radius), float(start_angle),
                                        1 if ccw else 0, float(sampling_ratio), 1 if collapsed else 0, float(width_ratio),
                                        int(num_profiles), cap, _ptr(prof), _ptr(xl), _ptr(yl), C.byref(cnt)))
    c = cnt.value
    return prof[:c].copy(), xl[:c].copy(), yl[:c].copy()


def single_profile(ctx: Context, values, params: SpParams, *, fwxm_x=50.0, penumbra=(20.0, 80.0), in_field_ratio=0.8,
                   slope_exclusion_ratio=0.2, x_values=None):
    """SingleProfile(values, ...) + every query method in one launch -> (result row, values, field values)."""
    v = np.ascontiguousarray(values, dtype=np.float64)
    n0 = v.size
    if params.interpolation == 1:
        n = int(round(n0 / (params.dpmm * params.interpolation_resolution_mm))) if params.dpmm > 0 else int(round(n0 * params.interpolation_factor))
    else:
        n = n0
    gw, lw = (gaussian_kernel1d(params.edge_smoothing_ratio * n) if params.edge == 1 else (None, 0))
    res = np.zeros(1, SP_RESULT_DTYPE)
    cap = n + 8
    vals, fv = np.empty(cap), np.empty(cap)
    xv = None if x_values is None else np.ascontiguousarray(x_values, dtype=np.float64)
    if xv is not None and xv.size != n0:
        raise ValueError("x_values and values must have the same length")
    check(lib().epid_single_profile(ctx.handle, _ptr(v), _ptr(xv), n0, C.byref(params), _ptr(gw), lw, n, float(fwxm_x), float(penumbra[0]),
                                    float(penumbra[1]), float(in_field_ratio), float(slope_exclusion_ratio), _ptr(res), _ptr(vals),
                                    _ptr(fv), cap))
    r = res[0]
    return r, vals[: int(r["n"])].copy(), fv[: int(r["fd_field_values_n"])].copy()
