"""QuasarLightRadScaling -- drop-in for ``pylinac.contrib.quasar`` (contrib/quasar.py:1-66): light/rad with BBs offset inward from
the measured field corners, and the five scaling BBs in a 35 mm window about the image centre, located in the same device call as
the rest of the analysis (csrc/lightrad.cu)."""
from __future__ import annotations

from ..core.geometry import Point
from ..planar_imaging import _SET_QUASAR, StandardImagingFC2


class QuasarLightRadScaling(StandardImagingFC2):
    """A light/rad and also scaling analysis for the Quasar phantom (contrib/quasar.py:6-66)."""

    common_name = "Quasar Light/Rad Scaling"
    bb_sampling_box_size_mm = 10
    bb_size_mm = 5
    field_strip_width_mm = 20
    light_rad_bb_offset_mm = 11
    scaling_centers: list[Point]
    _scaling_search = True

    @classmethod
    def _device_bb_set(cls):
        # _determine_bb_set: positions from the measured field widths, computed on the device; the keys are the reference's
        return {"TL": (0, 0), "BL": (0, 0), "TR": (0, 0), "BR": (0, 0)}, _SET_QUASAR

    def analyze(self, invert: bool = False, fwxm: int = 50, bb_edge_threshold_mm: float = 10) -> None:
        """Analyze the image for the light/rad and scaling"""
        super().analyze(invert=invert, fwxm=fwxm, bb_edge_threshold_mm=bb_edge_threshold_mm)
        self.scaling_centers = self._frame.scaling_centers
