"""Test helper: seeded Varian machine logs in the layouts the reference's log analyzer reads (log_analyzer.py:1764-1894, 2176-2336).

Trajectory log (.bin): a 1024-byte header ("VOSTL" and the version as 16-byte strings, header_size, sampling_interval, num_axes,
axis_enum[num_axes], samples_per_axis[num_axes] -- the MLC axis last, with leaves + 2 carriages --, axis_scale, num_subbeams,
is_truncated, num_snapshots, mlc_model; from v4.0 a 745-byte metadata block), one record per subbeam (int control point, float MU,
float radiation time, int sequence number, a 32-byte name before v3.0 or a 512-byte name from v3.0, then 32 reserved bytes) and the
body: num_snapshots x sum(samples_per_axis) x (expected, actual) float32 values.

Dynalog: an A / B pair of text files, 6 header lines then one comma-separated row of integers per snapshot: MU (or the gantry angle
for VMAT), previous segment, beam hold, beam on, prior / next dose index, gantry and collimator (0.1 deg), jaws Y1 Y2 X1 X2 (mm),
carriages A / B (0.01 mm) and per leaf of the file's bank (expected, actual, previous, next) in 0.01 mm at the MLC plane.
"""
from __future__ import annotations

import os
import struct

import numpy as np

N_PAIRS = 60


# ------------------------------------------------------------------------------------------------ trajectory logs
def tlog_axes(version: float) -> list[str]:
    """single-sample axes before the MLC, in file order (pitch / roll from v3.0)"""
    axes = ["collimator", "gantry", "y1", "y2", "x1", "x2", "vrt", "lng", "lat", "rtn"]
    if version >= 3:
        axes += ["pitch", "roll"]
    return axes + ["mu", "beam_hold", "control_point"]


def vmat_delivery(nsnap: int, seed: int, *, leaf_cm: float = 19.5, jaw_x: float = 6.0, jaw_y: float = 10.0, static_pairs=(),
                  crossed_pairs=(), mu_total: float = 150.0, holds: int = 0, gantry_rotates: bool = True, ncp: int = 50):
    """Columns of a synthetic VMAT-like beam (cm / deg / MU): dict of (expected, actual) float64 arrays per axis and 'leaves' as
    (expected, actual) arrays [nsnap, 2 * N_PAIRS] (bank A = leaves 1..60, bank B = 61..120, positive = open)."""
    rng = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, nsnap)
    cols = {}
    hold = np.zeros(nsnap)
    for k in range(holds):
        s0 = int(rng.integers(nsnap // 8, nsnap - nsnap // 8))
        hold[s0 : s0 + int(rng.integers(3, max(4, nsnap // 40)))] = 2
    mu_e = mu_total * t
    dmu = np.diff(mu_e, prepend=0.0)
    dmu[hold > 0] = 0.0
    mu_e = np.cumsum(dmu)
    mu_a = np.maximum.accumulate(mu_e + rng.normal(0, 0.002 * max(mu_total, 1e-3), nsnap))
    cols["mu"] = (mu_e, mu_a)
    cols["beam_hold"] = (hold, hold)
    cp = np.floor(t * (ncp - 1) + 1e-9)
    cols["control_point"] = (cp, cp)
    g = 181.0 + 358.0 * t if gantry_rotates else np.full(nsnap, 90.0)
    cols["gantry"] = (g, g + rng.normal(0, 0.02, nsnap))
    cols["collimator"] = (np.full(nsnap, 30.0), np.full(nsnap, 30.0) + rng.normal(0, 0.001, nsnap))
    for name, v in (("x1", jaw_x), ("x2", jaw_x + 1.0), ("y1", jaw_y), ("y2", jaw_y - 0.5)):
        e = np.full(nsnap, v) + 0.5 * np.sin(6.0 * t + len(name))
        cols[name] = (e, e + rng.normal(0, 0.003, nsnap))
    for name in ("vrt", "lng", "lat", "rtn", "pitch", "roll"):
        e = np.full(nsnap, float(rng.uniform(-5, 5)))
        cols[name] = (e, e + rng.normal(0, 0.001, nsnap))
    pairs = np.arange(N_PAIRS)
    phase = rng.uniform(0, 2 * np.pi, N_PAIRS)
    centre = leaf_cm * 0.6 * np.sin(2 * np.pi * (t[:, None] * 1.3 + phase[None, :] / 7))
    gap = 0.5 + 2.0 * np.abs(np.sin(3.0 * t[:, None] + phase[None, :]))
    a_e = centre + gap / 2                                   # bank A: right edge  (+x)
    b_e = -centre + gap / 2                                  # bank B: left edge   (-x, stored as a positive opening)
    a_e = np.clip(a_e, -leaf_cm, leaf_cm + 6.0)
    b_e = np.clip(b_e, -leaf_cm, leaf_cm + 6.0)
    for p in static_pairs:
        a_e[:, p] = 1.0 + 0.1 * p
        b_e[:, p] = 2.0 - 0.05 * p
    for p in crossed_pairs:
        a_e[:, p] = -1.5 - 0.5 * t
        b_e[:, p] = 0.7
    exp = np.concatenate([a_e, b_e], axis=1)
    noise = rng.normal(0, 0.004, exp.shape)
    noise[:, list(static_pairs) + [N_PAIRS + p for p in static_pairs]] = 0.0
    cols["leaves"] = (exp, exp + noise)
    cols["carriage_A"] = (np.full(nsnap, 10.0), np.full(nsnap, 10.0))
    cols["carriage_B"] = (np.full(nsnap, -10.0), np.full(nsnap, -10.0))
    del pairs
    return cols


def _str(s: str, n: int) -> bytes:
    b = s.encode("ascii")
    return b + b"\x00" * (n - len(b))


def tlog_bytes(cols, *, version: float = 3.0, mlc_model: int = 2, subbeams=((0, "Arc 1"),), metadata=None, truncate_body: int = 0,
               num_axes_override: int | None = None) -> bytes:
    """A trajectory log from `cols` (vmat_delivery).  subbeams: (control point, name) per subbeam; metadata (v4.0): dict."""
    axes = tlog_axes(version)
    nsnap = len(cols["mu"][0])
    nleaf = cols["leaves"][0].shape[1]
    num_axes = len(axes) + 1
    samples = [1] * len(axes) + [nleaf + 2]
    h = bytearray()
    h += _str("VOSTL", 16) + _str(f"{version:.1f}", 16)
    h += struct.pack("<iii", 1024, 20, num_axes if num_axes_override is None else num_axes_override)
    h += struct.pack(f"<{num_axes}i", *range(num_axes)) + struct.pack(f"<{num_axes}i", *samples)
    h += struct.pack("<iiiii", 1, len(subbeams), 0, nsnap, mlc_model)
    if version >= 4:
        md = metadata or {}
        fields = [("Patient ID", md.get("patient_id", "PT-0001")), ("Plan Name", md.get("plan_name", "VMAT QA")),
                  ("SOP Instance UID", md.get("sop", "1.2.246.352.71.5.1")), ("MU Planned", md.get("mu_planned", "150.000")),
                  ("MU Remaining", md.get("mu_remaining", "0.000")), ("Energy", md.get("energy", "6X")),
                  ("Beam Name", md.get("beam_name", "Arc 1"))]
        text = "\r\n".join(f"{k}:\t{v}" for k, v in fields) + "\r\n"
        h += _str(text, 745)
    h += b"\x00" * (1024 - len(h))
    chars = 512 if version >= 3 else 32
    for k, (cp, name) in enumerate(subbeams):
        h += struct.pack("<iffi", int(cp), float(np.float32(cols["mu"][0][-1] / max(len(subbeams), 1))), 12.5, k)
        h += _str(name, chars) + b"\x00" * 32
    body = np.empty((nsnap, sum(samples), 2), np.float32)
    for i, name in enumerate(axes):
        body[:, i, 0], body[:, i, 1] = cols[name]
    m0 = len(axes)
    body[:, m0, 0], body[:, m0, 1] = cols["carriage_A"]
    body[:, m0 + 1, 0], body[:, m0 + 1, 1] = cols["carriage_B"]
    body[:, m0 + 2 :, 0], body[:, m0 + 2 :, 1] = cols["leaves"]
    data = bytes(h) + body.tobytes()
    return data[: len(data) - truncate_body] if truncate_body else data


def write_tlog(path, cols, txt: dict | None = None, **kw) -> str:
    with open(path, "wb") as f:
        f.write(tlog_bytes(cols, **kw))
    if txt is not None:
        with open(str(path).replace(".bin", ".txt"), "w", encoding="utf-8") as f:
            for k, v in txt.items():
                f.write(f"{k}: {v}\n")
    return str(path)


# ------------------------------------------------------------------------------------------------ Dynalogs
DLG_CONV = 1.96078 / 1000


def dlog_rows(cols, *, vmat: bool = False, beam_off=()):
    """integer rows (A bank, B bank) from `cols` (vmat_delivery); MU as a dose fraction ending at 25000 or, for VMAT, the gantry angle"""
    nsnap = len(cols["mu"][0])
    mu = cols["mu"][1]
    if vmat:
        mucol = np.rint(cols["gantry"][1] * 10) % 3600
    else:
        mucol = np.rint(mu / mu[-1] * 25000) if mu[-1] > 0 else np.zeros(nsnap)
    beam_on = np.ones(nsnap)
    beam_on[list(beam_off)] = 0
    common = np.stack([mucol, np.arange(nsnap) // 10, cols["beam_hold"][1] > 0, beam_on, np.zeros(nsnap), np.zeros(nsnap),
                       np.rint(cols["gantry"][1] * 10), np.rint(cols["collimator"][1] * 10), np.rint(cols["y1"][1] * 10),
                       np.rint(cols["y2"][1] * 10), np.rint(cols["x1"][1] * 10), np.rint(cols["x2"][1] * 10),
                       np.full(nsnap, 5000), np.full(nsnap, -5000)], axis=1).astype(np.int64)
    banks = []
    for b in range(2):
        e = np.rint(cols["leaves"][0][:, b * N_PAIRS : (b + 1) * N_PAIRS] / DLG_CONV).astype(np.int64)
        a = np.rint(cols["leaves"][1][:, b * N_PAIRS : (b + 1) * N_PAIRS] / DLG_CONV).astype(np.int64)
        leaf = np.stack([e, a, e, e], axis=2).reshape(nsnap, -1)
        banks.append(np.concatenate([common, leaf], axis=1))
    return banks


def write_dlog_pair(directory, stem: str, cols, *, vmat: bool = False, beam_off=(), write_b: bool = True) -> tuple[str, str]:
    """A<stem>.dlg and B<stem>.dlg in `directory`; returns their paths"""
    paths = []
    for letter, rows in zip("AB", dlog_rows(cols, vmat=vmat, beam_off=beam_off)):
        p = os.path.join(str(directory), f"{letter}{stem}.dlg")
        paths.append(p)
        if letter == "B" and not write_b:
            continue
        lines = ["B", "PT0001,Doe^Jane", "plan.dat,1", "0", str(N_PAIRS), "0"] + [",".join(str(int(v)) for v in r) for r in rows]
        with open(p, "w", encoding="utf-8", newline="") as f:
            f.write("\r\n".join(lines) + "\r\n")
    return paths[0], paths[1]
