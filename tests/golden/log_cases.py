"""Seeded machine logs for tests/golden/log_golden.npz (make_log_golden.py runs the unmodified reference's log analyzer on them).

write_case(name, directory) writes the case's file(s) with tests/log_writer.py and returns the path to load.  The golden stores
each written file's sha1, so a change in the writer shows up as a golden mismatch rather than a silent new input."""
from __future__ import annotations

import os

from tests import log_writer as lw

# (fluence resolution, equal_aspect) pairs stored for every case with a fluence; 0.3 does not divide 5 mm
MAP_SETTINGS = ((0.1, False), (0.5, False), (1.0, False), (0.3, False), (0.5, True), (1.0, True), (0.3, True))
SUBBEAM_SETTINGS = ((0.5, False),)
# gamma settings: (doseTA, distTA, threshold, resolution)
GAMMA_SETTINGS = ((1, 1, 0.1, 0.1), (2, 2, 0.2, 0.5))
SUB_ROWS, SUB_COLS = slice(None, None, 7), slice(None, None, 13)      # subsample of the stored maps (plus a sha1 of the whole map)

CASES = ("tlog_v21_millennium", "tlog_v30_hd_subbeams", "tlog_v40_metadata", "tlog_static", "tlog_no_mu", "dlog_regular", "dlog_vmat")
BAD_CASES = ("tlog_no_subbeams", "tlog_truncated", "tlog_bad_version", "tlog_bad_metadata", "dlog_without_b", "not_a_log")


def write_case(name: str, directory) -> str:
    d = str(directory)
    if name == "tlog_v21_millennium":
        cols = lw.vmat_delivery(700, 1, holds=2)
        return lw.write_tlog(os.path.join(d, "PT1_v21.bin"), cols, version=2.1, txt={"Patient ID": "PT1", "Plan Name": "VMAT QA"})
    if name == "tlog_v30_hd_subbeams":
        cols = lw.vmat_delivery(900, 2, leaf_cm=21.0, jaw_y=4.0, static_pairs=(3, 30, 44), crossed_pairs=(25, 27), holds=1)
        return lw.write_tlog(os.path.join(d, "PT2_v30.bin"), cols, version=3.0, mlc_model=3,
                             subbeams=((0, "Arc 1"), (18, "Arc 2"), (35, "Arc 3")))
    if name == "tlog_v40_metadata":
        cols = lw.vmat_delivery(800, 3, jaw_x=20.5, jaw_y=11.0, crossed_pairs=(31,), mu_total=25000.0)
        return lw.write_tlog(os.path.join(d, "PT3_v40.bin"), cols, version=4.0, subbeams=((0, "Arc 1"), (20, "Arc 2")),
                             metadata={"patient_id": "PT3", "beam_name": "Arc 1"})
    if name == "tlog_static":
        cols = lw.vmat_delivery(400, 4, static_pairs=tuple(range(60)), gantry_rotates=False, jaw_y=6.0)
        return lw.write_tlog(os.path.join(d, "PT4_static.bin"), cols, version=3.0)
    if name == "tlog_no_mu":
        cols = lw.vmat_delivery(300, 5, mu_total=0.3, gantry_rotates=False)
        return lw.write_tlog(os.path.join(d, "PT5_nomu.bin"), cols, version=3.0, subbeams=((0, "Setup"), (25, "kV")))
    if name == "dlog_regular":
        cols = lw.vmat_delivery(600, 6, jaw_y=8.0, static_pairs=(12,), holds=2)
        return lw.write_dlog_pair(d, "PT6_regular", cols, beam_off=range(590, 600))[0]
    if name == "dlog_vmat":
        cols = lw.vmat_delivery(500, 7, crossed_pairs=(40,))
        return lw.write_dlog_pair(d, "PT7_vmat", cols, vmat=True)[1]
    if name == "tlog_no_subbeams":
        return lw.write_tlog(os.path.join(d, "PT8_nosub.bin"), lw.vmat_delivery(120, 8), version=3.0, subbeams=())
    if name == "tlog_truncated":
        return lw.write_tlog(os.path.join(d, "PT9_trunc.bin"), lw.vmat_delivery(120, 9), version=3.0, truncate_body=100)
    if name == "tlog_bad_version":
        p = lw.write_tlog(os.path.join(d, "PT10_badver.bin"), lw.vmat_delivery(50, 10), version=3.0)
        data = bytearray(open(p, "rb").read())
        data[16:32] = b"v3.x" + b"\x00" * 12
        open(p, "wb").write(bytes(data))
        return p
    if name == "tlog_bad_metadata":
        return lw.write_tlog(os.path.join(d, "PT11_badmeta.bin"), lw.vmat_delivery(50, 11), version=4.0,
                             metadata={"mu_planned": "lots"})
    if name == "dlog_without_b":
        return lw.write_dlog_pair(d, "PT12_alone", lw.vmat_delivery(50, 12), write_b=False)[0]
    if name == "not_a_log":
        p = os.path.join(d, "notes.bin")
        open(p, "wb").write(b"hello, this is not a machine log" * 4)
        return p
    raise KeyError(name)
