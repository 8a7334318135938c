"""Generate tests/golden/lightrad_golden.npz by running the UNMODIFIED reference light/rad phantom classes (planar_imaging.py:1169-1727,
contrib/quasar.py), stub-imported from the reference source tree (oracle/refstub.py), on the seeded synthetic cases of lightrad_cases.py.  skimage's
equalize_adapthist is served by tests/golden/clahe_restated.py, label, clear_border and regionprops by oracle/skimage_shim.py
(restated, unpinned at that boundary).

Run where the reference source tree is available:  python -m tests.golden.make_lightrad_golden
"""
from __future__ import annotations

import hashlib
import sys
import warnings

import numpy as np

from tests.golden.lightrad_cases import CASES, lightrad_case


def reference_lightrad(cls_name, frame, dpmm, ctor, analyze):
    from tests.golden import clahe_restated

    clahe_restated.install()
    import pylinac.contrib.quasar as rq
    import pylinac.planar_imaging as rp

    cls = rq.QuasarLightRadScaling if cls_name == "QuasarLightRadScaling" else getattr(rp, cls_name)
    out = {}
    near = []
    orig = rp.StandardImagingFC2._is_bb_near_edge

    def spy(self, bb_position):              # observe (not alter) the near-edge decisions in visiting order
        r = orig(self, bb_position)
        near.append(bool(r))
        return r

    rp.StandardImagingFC2._is_bb_near_edge = spy
    try:
        ph = cls(np.array(frame), image_kwargs=dict(dpi=25.4 * dpmm), **ctor)
        out["dpmm"] = float(ph.image.dpmm)
        ph.analyze(**analyze)
    except Exception as e:                   # noqa: BLE001 - the exception type and message are part of the golden
        out["error_type"] = np.array(type(e).__name__)
        out["error_message"] = np.array(str(e))
        return out
    finally:
        rp.StandardImagingFC2._is_bb_near_edge = orig
    out["field_center"] = np.array([ph.field_center.x, ph.field_center.y], dtype=float)
    out["field_width"] = np.array([ph.field_width_x, ph.field_width_y], dtype=float)
    out["bb_center"] = np.array([ph.bb_center.x, ph.bb_center.y], dtype=float)
    out["bb_keys"] = np.array(list(ph.bb_centers.keys()))
    out["bb_centers"] = np.array([[p.x, p.y] for p in ph.bb_centers.values()], dtype=float)
    out["epid_center"] = np.array([ph.epid_center.x, ph.epid_center.y], dtype=float)
    out["field_epid_offset_mm"] = np.array([ph.field_epid_offset_mm.x, ph.field_epid_offset_mm.y], dtype=float)
    out["field_bb_offset_mm"] = np.array([ph.field_bb_offset_mm.x, ph.field_bb_offset_mm.y], dtype=float)
    out["near_edge"] = np.array(near, dtype=bool)
    # an ArrayImage has no `source`, which the reference's "File:" line reads (core/image.py:498-512): give it an empty one
    ph.image.source, ph.image.path = "", ""
    out["results"] = np.array(ph.results(as_list=True))
    rd = ph.results_data()
    out["results_data"] = np.array([rd.field_size_x_mm, rd.field_size_y_mm, rd.field_epid_offset_x_mm, rd.field_epid_offset_y_mm,
                                    rd.field_bb_offset_x_mm, rd.field_bb_offset_y_mm], dtype=float)
    if hasattr(ph, "scaling_centers"):
        out["scaling_centers"] = np.array([[p.x, p.y] for p in ph.scaling_centers], dtype=float)
    return out


def main():
    store = {}
    warnings.simplefilter("ignore")
    for name in CASES:
        c = lightrad_case(name)
        store[f"{name}/input_sha1"] = np.frombuffer(hashlib.sha1(c["frame"].tobytes()).digest(), dtype=np.uint8)
        ref = reference_lightrad(c["cls"], c["frame"], c["dpmm"], c["ctor"], c["analyze"])
        for k, v in ref.items():
            store[f"{name}/{k}"] = np.asarray(v)
        for k, v in c["truth"].items():
            store[f"{name}/truth_{k}"] = np.asarray(v)
        print(name, c["cls"], ref.get("error_type", ""), np.round(ref.get("field_width", np.zeros(2)), 3),
              ref.get("near_edge", ""), np.round(ref.get("field_bb_offset_mm", np.zeros(2)), 3))
    np.savez_compressed("tests/golden/lightrad_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
