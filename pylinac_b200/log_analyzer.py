"""Machine-log analysis: ``pylinac.log_analyzer`` (log_analyzer.py:54-2951) with the fluence maps and the fluence gamma on the GPU.

Parsing (trajectory-log header / subbeams / axis data, the Dynalog text and its A / B pair) and the MLC statistics are host work with
the reference's numpy expressions: they cost O(leaves x snapshots) and ``moving_leaves`` decides the fluence branch of every pair,
which must match the reference bit for bit.  ``FluenceBase.calc_map`` -- pairs x snapshots x columns -- runs in ``epid_log_fluence``
(csrc/logs.cu); ``GammaFluence.calc_map`` runs the device operators ``BaseImage.gamma`` uses (inversion check, ground, normalize,
``epid_gamma``) on the device-resident maps plus one per-frame reduction for ``avg_gamma`` / ``pass_prcnt``.  Fluence and gamma
maps stay on the device until a caller reads ``.array``.

Device input: every log is a column table in one host arena (csrc/logs.cu): a trajectory log's raw float32 body as read from the
file (the kernel widens to fp64, as the reference's ``decode_binary`` does), a Dynalog's fp64 columns (text integers x
(1.96078 / 1000) for the leaves, the corrected MU, the jaws in cm) built on the host.

Not included (as for the other modules): plots, PDF, ``to_csv``, ``anonymize``, ``from_url``, ``from_demo``.
"""
from __future__ import annotations

import copy
import csv
import enum
import itertools
import os
import os.path as osp
import struct
import tempfile
import zipfile
from collections.abc import Iterable, Sequence
from dataclasses import dataclass
from functools import cached_property

import numpy as np

from . import _native as nat
from .core.utilities import convert_to_enum


class TreatmentType(enum.Enum):  # log_analyzer.py:54-58
    STATIC_IMRT = "Static IMRT"
    DYNAMIC_IMRT = "Dynamic IMRT"
    VMAT = "VMAT"
    IMAGING = "Imaging"


MLC_FOV_WIDTH_MM = 400
MLC_FOV_HEIGHT_MM = 400
HDMLC_FOV_HEIGHT_MM = 220


class MLCBank(enum.Enum):  # :66-69
    A = "A"
    B = "B"
    BOTH = "both"


class Fluence(enum.Enum):  # :72-75
    ACTUAL = "actual"
    EXPECTED = "expected"
    GAMMA = "gamma"


class NotALogError(IOError):  # :2934-2937
    """The passed file is not a valid machine log file."""


class NotADynalogError(IOError):  # :2940-2943
    """The passed file is not a valid Dynalog file."""


class DynalogMatchError(IOError):  # :2946-2951
    """The companion file of a Dynalog (A file for a B file and vice versa) was not found."""


# ------------------------------------------------------------------------------------------------ decode_binary (core/utilities.py:232-288)
def _take(f, n: int) -> bytes:
    b = f.read(n)
    if len(b) != n:
        raise struct.error(f"unpack requires a buffer of {n} bytes")
    return b


def _ints(f, count: int = 1):
    vals = np.asarray(struct.unpack("i" * count, _take(f, 4 * count)))
    return int(np.squeeze(vals)) if len(vals) == 1 else vals


def _floats(f, count: int = 1):
    vals = np.asarray(struct.unpack("f" * count, _take(f, 4 * count)))
    return float(np.squeeze(vals)) if len(vals) == 1 else vals


def _text(f, count: int, cursor_shift: int = 0) -> str:
    # one byte at a time, NULs dropped: a byte >= 0x80 raises UnicodeDecodeError as in the reference
    s = "".join(bytes([b]).decode() for b in _take(f, count) if b != 0)
    if cursor_shift:
        f.seek(cursor_shift, 1)
    return s


# ------------------------------------------------------------------------------------------------ axes (:315-437)
class Axis:
    """actual and (optionally) expected positions of one axis"""

    def __init__(self, actual: np.ndarray, expected: np.ndarray | None = None):
        self.actual = actual
        self.expected = expected
        if expected is not None:
            try:
                if len(actual) != len(expected):
                    raise ValueError("Actual and expected Axis parameters are not equal length")
            except TypeError:
                pass

    @property
    def difference(self) -> np.ndarray:
        if self.expected is not None:
            return self.actual - self.expected
        raise AttributeError("Expected positions not passed to Axis")


class AxisMovedMixin:
    AXIS_MOVE_THRESHOLD: float = 0.003

    @cached_property
    def moved(self) -> bool:
        return np.std(self.actual) > self.AXIS_MOVE_THRESHOLD


class LeafAxis(Axis, AxisMovedMixin):
    def __init__(self, actual, expected):
        super().__init__(actual, expected)


class GantryAxis(Axis, AxisMovedMixin):
    pass


class HeadAxis(Axis, AxisMovedMixin):
    pass


class CouchAxis(Axis, AxisMovedMixin):
    pass


class BeamAxis(Axis):
    pass


class JawStruct:  # :1351-1375
    def __init__(self, x1: HeadAxis, y1: HeadAxis, x2: HeadAxis, y2: HeadAxis):
        if not all(isinstance(a, HeadAxis) for a in (x1, y1, x2, y2)):
            raise TypeError("HeadAxis not passed into Jaw structure")
        self.x1, self.y1, self.x2, self.y2 = x1, y1, x2, y2


class CouchStruct:  # :1378-1415
    def __init__(self, vertical: CouchAxis, longitudinal: CouchAxis, lateral: CouchAxis, rotational: CouchAxis,
                 pitch: CouchAxis | None = None, roll: CouchAxis | None = None):
        if not all(isinstance(a, CouchAxis) for a in (vertical, longitudinal, lateral, rotational)):
            raise TypeError("Couch structure must be passed Couch Axes.")
        self.vert, self.long, self.latl, self.rotn = vertical, longitudinal, lateral, rotational
        self.pitch, self.roll = (pitch, roll) if pitch is not None else (None, None)


# ------------------------------------------------------------------------------------------------ device column tables
class _Source:
    """Where a log's fluence inputs sit in a host buffer (see the module docstring): `buf` is a float32 [nsnap, 2 * sum(samples)]
    trajectory-log body or a float64 [columns, nsnap] Dynalog table; columns are (actual, expected) of MU, X1 / X2 actual and the
    leaf-1 column of each kind (leaf l at + 2 (l - 1))."""

    def __init__(self, buf: np.ndarray, col_mu, col_x1: int, col_x2: int, col_leaf):
        self.buf = buf
        self.col_mu, self.col_x1, self.col_x2, self.col_leaf = tuple(col_mu), col_x1, col_x2, tuple(col_leaf)

    @property
    def f64(self) -> bool:
        return self.buf.dtype == np.float64

    @property
    def nsnap(self) -> int:
        return self.buf.shape[1] if self.f64 else self.buf.shape[0]

    @property
    def strides(self) -> tuple[int, int]:   # (snapshot, column) in elements
        return (1, self.buf.shape[1]) if self.f64 else (self.buf.shape[1], 1)

    @classmethod
    def from_axes(cls, mlc, mu: Axis, jaws: JawStruct) -> "_Source":
        """fp64 column table of any MLC / MU / jaw structure (the values the reference's calc_map reads)"""
        cols = [np.asarray(mu.actual, np.float64), np.asarray(mu.expected if mu.expected is not None else mu.actual, np.float64),
                np.asarray(jaws.x1.actual, np.float64), np.asarray(jaws.x2.actual, np.float64)]
        for leaf in range(1, mlc.num_leaves + 1):
            cols += [np.asarray(mlc.leaf_axes[leaf].expected, np.float64), np.asarray(mlc.leaf_axes[leaf].actual, np.float64)]
        return cls(np.ascontiguousarray(np.stack(cols)), (0, 1), 2, 3, (5, 4))


def _slot(nbytes: int) -> int:
    return (nbytes + 15) & ~15


def _arena(sources: list[_Source], pinned: bool):
    """-> (uint8 arena, byte offset of every source).  Sources that already live in one buffer are used in place: only the byte span
    that holds them is handed over (and copied to the device), not the whole shared buffer."""
    bases = {id(getattr(s.buf, "_arena", None)) for s in sources}
    if len(bases) == 1 and getattr(sources[0].buf, "_arena", None) is not None:
        arena = sources[0].buf._arena
        base = arena.ctypes.data
        lo = min(s.buf.ctypes.data for s in sources) - base
        hi = max(s.buf.ctypes.data + s.buf.nbytes for s in sources) - base
        return np.asarray(arena[lo:hi]), [s.buf.ctypes.data - base - lo for s in sources]
    if len(sources) == 1:
        return sources[0].buf.reshape(-1).view(np.uint8), [0]
    offs, pos = [], 0
    for s in sources:
        offs.append(pos)
        pos += _slot(s.buf.nbytes)
    arena = nat.pinned_empty((max(pos, 16),), np.uint8) if pinned else np.empty(max(pos, 16), np.uint8)
    for s, o in zip(sources, offs):
        arena[o : o + s.buf.nbytes] = s.buf.reshape(-1).view(np.uint8)
    return arena, offs


class _Maps:
    """a device batch of maps shared by several fluence objects; downloaded once on the first host read"""

    def __init__(self, batch: nat.Batch):
        self.batch = batch
        self._host = None

    def host(self) -> np.ndarray:
        if self._host is None:
            self._host = self.batch.download()
        return self._host


def _leaf_rows(hdmlc: bool, resolution: float) -> np.ndarray:
    """create_mlc_y_positions (:522-543): leaf boundaries in pixel rows, a float cumsum cast to int"""
    if not hdmlc:
        n_large, s_large, n_small, s_small = 10, 10 / resolution, 40, 5 / resolution
    else:
        n_large, s_large, n_small, s_small = 14, 5 / resolution, 32, 2.5 / resolution
    sizes = [s_large] * n_large + [s_small] * n_small + [s_large] * n_large
    return np.cumsum([0] + sizes).astype(int)


def _fluence_rows(fl: "FluenceBase", resolution: float, equal_aspect: bool) -> int:
    height = MLC_FOV_HEIGHT_MM if not fl._mlc.hdmlc else HDMLC_FOV_HEIGHT_MM
    return int(height / resolution) if equal_aspect else fl._mlc.num_pairs


@dataclass
class _FluenceInputs:
    """everything one epid_log_fluence launch reads, built on the host"""

    arena: np.ndarray
    descs: np.ndarray
    snaps: np.ndarray
    pair_flags: np.ndarray
    rows: np.ndarray
    resolution: float
    W: int
    R: int
    kinds: int

    def launch(self, ctx=None):
        """-> the (actual, expected) _Maps (None for a kind not requested)"""
        a, e = nat.log_fluence(ctx or nat.Context.default(), self.arena, self.descs, self.snaps, self.pair_flags, self.rows,
                               self.resolution, self.W, self.R, self.kinds)
        return (_Maps(a) if a is not None else None), (_Maps(e) if e is not None else None)


def _compute_fluences(items, resolution: float, equal_aspect: bool, kinds: int = 3, pinned: bool = True, ctx=None):
    """epid_log_fluence for `items` = [(FluenceStruct-like with .actual / .expected, _Source)], all of one map shape.
    Returns the (actual, expected) _Maps (None for a kind not requested)."""
    return _fluence_inputs(items, resolution, equal_aspect, kinds, pinned).launch(ctx)


def _fluence_inputs(items, resolution: float, equal_aspect: bool, kinds: int = 3, pinned: bool = True) -> _FluenceInputs:
    """the host half of _compute_fluences: descriptors, beam-on lists, the reference's per-pair decisions, row bounds, the arena"""
    W = int(MLC_FOV_WIDTH_MM / resolution)
    R = _fluence_rows(items[0][0].actual, resolution, equal_aspect)
    descs = np.zeros(len(items), nat.LOG_DESC_DTYPE)
    snaps, pflags, rows = [], [], []
    n_snaps = n_pf = n_rows = 0
    for i, (fs, src) in enumerate(items):
        fl = fs.actual
        mlc = fl._mlc
        if _fluence_rows(fl, resolution, equal_aspect) != R:
            raise ValueError("every log of one fluence launch must have the same map shape")
        d = descs[i]
        d["snap_stride"], d["col_stride"] = src.strides
        d["f64"], d["nsnap"] = int(src.f64), src.nsnap
        d["col_mu"], d["col_x1"], d["col_x2"], d["col_leaf"] = src.col_mu, src.col_x1, src.col_x2, src.col_leaf
        d["num_pairs"] = mlc.num_pairs
        sidx = np.asarray(mlc.snapshot_idx, dtype=np.int64).reshape(-1)
        flags = [0, 0]
        for k, attr in enumerate(("actual", "expected")):
            mu = getattr(fl._mu, attr)
            if len(mlc.snapshot_idx) < 1 or np.max(mu) < 0.5:
                flags[k] = nat.LF_ZERO
            elif mu[-1] == 25000:
                flags[k] = nat.LF_DIV25000
        d["flags"] = flags
        live = [k for k in range(2) if (kinds >> k) & 1 and not flags[k] & nat.LF_ZERO]
        if live:
            positions = _leaf_rows(mlc.hdmlc, resolution)
            if mlc.num_pairs + 1 > len(positions):     # the reference's leaf-width generator runs past its table
                raise IndexError(f"index {len(positions)} is out of bounds for axis 0 with size {len(positions)}")
        d["snap_off"], d["nbeam"] = n_snaps, (len(sidx) if live else 0)
        if live:
            snaps.append(sidx.astype(np.int32))
            n_snaps += len(sidx)
        pf = np.zeros(mlc.num_pairs, np.uint8)
        rb = np.zeros((mlc.num_pairs, 2), np.int32)
        if live:
            for pair in range(1, mlc.num_pairs + 1):
                if mlc.leaf_under_y_jaw(pair):
                    pf[pair - 1] = nat.PF_UNDER_JAW
                    continue
                if mlc.pair_moved(pair):
                    pf[pair - 1] = nat.PF_MOVED
                if equal_aspect:
                    rb[pair - 1] = [min(positions[pair - 1], R), min(positions[pair], R)]
                else:
                    rb[pair - 1] = [pair - 1, pair]
        d["pair_off"], d["row_off"] = n_pf, n_rows
        pflags.append(pf)
        rows.append(rb.reshape(-1))
        n_pf += len(pf)
        n_rows += rb.size
    arena, offs = _arena([src for _, src in items], pinned)
    descs["data_off"] = offs
    cat = lambda parts, dt: np.concatenate(parts).astype(dt) if parts else np.zeros(0, dt)  # noqa: E731
    return _FluenceInputs(arena, descs, cat(snaps, np.int32), cat(pflags, np.uint8), cat(rows, np.int32), resolution, W, R, kinds)


def _gamma_maps(actual: nat.Batch, expected: nat.Batch, doseTA, distTA, threshold, resolution, ctx=None):
    """BaseImage.gamma (core/image.py:928-1017) of every (actual, expected) frame pair on the device -> (gamma Batch, avg, pct)"""
    if not 0.0 <= threshold <= 1.0:
        raise ValueError("threshold must be between 0 and 1")
    ctx = ctx or nat.Context.default()
    lib = nat.lib()

    def prepared(b: nat.Batch) -> nat.Batch:
        h = nat._P()
        with nat.hist_invert(ctx, b)[0] as inv:
            nat.check(lib.epid_ground(ctx.handle, inv.handle, 0.0, nat.C.byref(h), None))
        with nat.Batch(ctx, h) as grounded:
            return grounded._unary(lib.epid_normalize, 1, 0.0)

    with prepared(actual) as ref, prepared(expected) as comp:
        # after normalize() the reference's max is exactly 1.0 (or nan for a constant map, where every pixel is nan already)
        dpmm = (25.4 / resolution) / 25.4
        g = ref._unary2(lib.epid_gamma, comp, float(threshold * 1.0), doseTA / 100.0, float(dpmm * distTA))
    s, cnt, passing = nat.gamma_stats(ctx, g)
    avg, pct = [], []
    with np.errstate(invalid="ignore", divide="ignore"):
        for k in range(len(s)):
            avg.append(np.float64(s[k] / cnt[k]) if cnt[k] else 0)              # np.nanmean, nan -> 0 (:743-745)
            pct.append(np.int64(passing[k]) / np.int64(cnt[k]) * 100)           # :746-748
    return g, avg, pct


# ------------------------------------------------------------------------------------------------ fluences (:439-841)
class FluenceBase:
    """A fluence map: num_pairs (or int(height / resolution)) x int(400 / resolution), float64, device-resident once computed."""

    resolution = -1
    FLUENCE_TYPE = ""

    def __init__(self, mlc_struct=None, mu_axis: Axis = None, jaw_struct=None, source: _Source | None = None):
        self._host = np.empty((0, 0))
        self._dev: tuple[_Maps, int] | None = None
        self._mlc = mlc_struct
        self._mu = mu_axis
        self._jaws = jaw_struct
        self._source = source
        self._key = None

    @property
    def array(self) -> np.ndarray:
        if self._dev is not None:
            maps, i = self._dev
            return maps.host()[i]
        return self._host

    @array.setter
    def array(self, value) -> None:
        self._host = value
        self._dev = None
        self._key = None

    def is_map_calced(self, raise_error: bool = False) -> bool:
        calced = self._dev is not None or self._host.size > 0
        if not calced and raise_error:
            raise ValueError("Map has not yet been calculated. Use .calc_map() with desired parameters first.")
        return calced

    def _struct(self):
        return _Pair(self._mlc, self._mu, self._jaws)

    def _src(self) -> _Source:
        if self._source is None:
            self._source = _Source.from_axes(self._mlc, self._mu, self._jaws)
        return self._source

    def _set(self, maps: _Maps, i: int, resolution, key) -> None:
        self._dev = (maps, i)
        self._host = np.empty((0, 0))
        self.resolution = resolution
        self._key = key

    def calc_map(self, resolution: float = 0.1, equal_aspect: bool = False) -> np.ndarray:
        """The fluence map (log_analyzer.py:478-612), computed on the device (epid_log_fluence)."""
        key = (resolution, equal_aspect)
        if self._key != key or self._dev is None:
            kind = 1 if self.FLUENCE_TYPE == "actual" else 2
            a, e = _compute_fluences([(self._struct(), self._src())], resolution, equal_aspect, kinds=kind, pinned=False)
            self._set(a if kind == 1 else e, 0, resolution, key)
        return self.array


class _Pair:
    """the (actual, expected) view _compute_fluences reads: both share the MLC / MU / jaws of one fluence"""

    def __init__(self, mlc, mu, jaws):
        self.actual = FluenceBase(mlc, mu, jaws)


class ActualFluence(FluenceBase):
    FLUENCE_TYPE = "actual"


class ExpectedFluence(FluenceBase):
    FLUENCE_TYPE = "expected"


class GammaFluence(FluenceBase):
    """Gamma map of the actual against the expected fluence (log_analyzer.py:640-822)."""

    distTA = -1
    doseTA = -1
    threshold = -1
    pass_prcnt = -1
    avg_gamma = -1
    bins = [0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1, 1.1]

    def __init__(self, actual_fluence: ActualFluence, expected_fluence: ExpectedFluence, mlc_struct):
        super().__init__(mlc_struct)
        self._actual_fluence = actual_fluence
        self._expected_fluence = expected_fluence

    @property
    def array(self) -> np.ndarray:
        if self._dev is not None:
            maps, i = self._dev
            return np.nan_to_num(maps.host()[i])
        return self._host

    @array.setter
    def array(self, value) -> None:
        self._host = value
        self._dev = None
        self._key = None

    @property
    def passfail_array(self) -> np.ndarray:
        return self.array >= 1

    def _finish(self, maps: _Maps, i: int, avg, pct, doseTA, distTA, threshold, resolution) -> None:
        self._set(maps, i, resolution, (doseTA, distTA, threshold, resolution))
        self.avg_gamma, self.pass_prcnt = avg, pct
        self.distTA, self.doseTA, self.threshold = distTA, doseTA, threshold

    def calc_map(self, doseTA: float = 1, distTA: float = 1, threshold: float = 0.1, resolution: float = 0.1,
                 calc_individual_maps: bool = False) -> np.ndarray:
        key = (doseTA, distTA, threshold, resolution)
        if self._key == key and self._dev is not None:
            return self.array
        for fl in (self._actual_fluence, self._expected_fluence):
            if not fl.is_map_calced() or resolution != fl.resolution:
                fl.calc_map(resolution)
        a, e = self._actual_fluence, self._expected_fluence
        if _map_shape(a) != _map_shape(e):
            raise AttributeError(f"The images are not the same size: {_map_shape(a)} vs. {_map_shape(e)}")
        ctx = nat.Context.default()
        ba = _single_batch(ctx, a)
        be = _single_batch(ctx, e)
        try:
            g, avg, pct = _gamma_maps(ba, be, doseTA, distTA, threshold, resolution, ctx)
        finally:
            for b, fl in ((ba, a), (be, e)):
                if fl._dev is None or b is not fl._dev[0].batch:
                    b.free()
        self._finish(_Maps(g), 0, avg[0], pct[0], doseTA, distTA, threshold, resolution)
        return self.array

    def histogram(self, bins: list | None = None) -> tuple[np.ndarray, np.ndarray]:
        self.is_map_calced(raise_error=True)
        return np.histogram(self.array, bins=self.bins if bins is None else bins)


def _map_shape(fl: FluenceBase) -> tuple:
    return fl._dev[0].batch.shape_dtype[0][1:] if fl._dev is not None else fl._host.shape


def _single_batch(ctx, fl: FluenceBase) -> nat.Batch:
    """a device batch holding just this fluence's map (the shared batch itself when it has one frame)"""
    if fl._dev is not None and fl._dev[0].batch.shape_dtype[0][0] == 1:
        return fl._dev[0].batch
    return nat.Batch.upload(ctx, np.ascontiguousarray(fl.array, dtype=np.float64)[None])


class FluenceStruct:  # :825-841
    def __init__(self, mlc_struct=None, mu_axis: Axis = None, jaw_struct=None, source: _Source | None = None):
        self.actual = ActualFluence(mlc_struct, mu_axis, jaw_struct, source)
        self.expected = ExpectedFluence(mlc_struct, mu_axis, jaw_struct, source)
        self.gamma = GammaFluence(self.actual, self.expected, mlc_struct)


# ------------------------------------------------------------------------------------------------ MLC (:844-1348)
class MLC:
    def __init__(self, log_type, snapshot_idx=None, jaw_struct=None, hdmlc: bool = False, subbeams=None):
        self.leaf_axes: dict = {}
        self.snapshot_idx = snapshot_idx
        self._jaws = jaw_struct
        self.hdmlc = hdmlc
        self.log_type = log_type
        self.subbeams = subbeams

    @classmethod
    def from_dlog(cls, dlog, jaws, snapshot_data: np.ndarray, snapshot_idx, b_snapshot_data: np.ndarray | None = None):
        mlc = MLC(Dynalog, snapshot_idx, jaws)
        half = dlog.header.num_mlc_leaves // 2
        for leaf in range(1, half + 1):
            mlc.add_leaf_axis(LeafAxis(expected=snapshot_data[(leaf - 1) * 4 + 14], actual=snapshot_data[(leaf - 1) * 4 + 15]), leaf)
        if b_snapshot_data is None:
            b_snapshot_data = _read_dlog_table(dlog.b_logfile)[1]
        for leaf in range(1, half + 1):
            mlc.add_leaf_axis(LeafAxis(expected=b_snapshot_data[(leaf - 1) * 4 + 14], actual=b_snapshot_data[(leaf - 1) * 4 + 15]),
                              leaf + half)
        # MLC plane -> isocentre plane and 0.01 mm -> cm (:917-925), in place like the reference
        for leaf in range(1, mlc.num_leaves + 1):
            mlc.leaf_axes[leaf].actual *= 1.96078 / 1000
            mlc.leaf_axes[leaf].expected *= 1.96078 / 1000
        return mlc

    @classmethod
    def from_tlog(cls, tlog, subbeams, jaws, snapshot_data, snapshot_idx, column_iter):
        mlc = MLC(TrajectoryLog, snapshot_idx, jaws, tlog.is_hdmlc, subbeams=subbeams)
        for leaf_num in range(1, tlog.header.num_mlc_leaves + 1):
            mlc.add_leaf_axis(_get_axis(snapshot_data, next(column_iter), LeafAxis), leaf_num)
        return mlc

    @property
    def num_pairs(self) -> int:
        return int(self.num_leaves / 2)

    @property
    def num_leaves(self) -> int:
        return len(self.leaf_axes)

    @property
    def num_snapshots(self) -> int:
        return len(self.snapshot_idx)

    @property
    def num_moving_leaves(self) -> int:
        return len(self.moving_leaves)

    @cached_property
    def moving_leaves(self) -> np.ndarray:
        """leaves whose actual-position std over snapshot_idx exceeds 0.01 cm (:962-974).  The reference's trajectory-log branch
        (std over the last subbeam's snapshots) tests ``isinstance(self, TrajectoryLog)`` on the MLC object and is never taken."""
        indices = ()
        for leaf_num, leafdata in self.leaf_axes.items():
            if np.std(leafdata.actual[self.snapshot_idx]) > 0.01:
                indices += (leaf_num,)
        return np.array(indices)

    def add_leaf_axis(self, leaf_axis: LeafAxis, leaf_num: int) -> None:
        self.leaf_axes[leaf_num] = leaf_axis

    def leaf_moved(self, leaf_num: int) -> bool:
        return leaf_num in self.moving_leaves

    def pair_moved(self, pair_num: int) -> bool:
        return self.leaf_moved(pair_num) or self.leaf_moved(pair_num + self.num_pairs)

    @property
    def _all_leaf_indices(self) -> np.ndarray:
        return np.array(range(1, len(self.leaf_axes) + 1))

    def get_RMS_avg(self, bank: MLCBank = MLCBank.BOTH, only_moving_leaves: bool = False):
        rms = np.mean(self.create_RMS_array(self.get_leaves(bank, only_moving_leaves)))
        return 0 if np.isnan(rms) else rms

    def get_RMS_max(self, bank: MLCBank = MLCBank.BOTH) -> float:
        rms = np.max(self.create_RMS_array(self.get_leaves(bank)))
        return 0 if np.isnan(rms) else rms

    def get_RMS_percentile(self, percentile: float = 95, bank: MLCBank = MLCBank.BOTH, only_moving_leaves: bool = False):
        return np.percentile(self.create_RMS_array(self.get_leaves(bank, only_moving_leaves)), percentile)

    def get_RMS(self, leaves_or_bank) -> np.ndarray:
        if isinstance(leaves_or_bank, (str, MLCBank)):
            leaves_or_bank = self.get_leaves(leaves_or_bank)
        elif not isinstance(leaves_or_bank, Iterable):
            raise TypeError("Input must be iterable, or specify an MLC bank")
        return self.create_RMS_array(np.array(leaves_or_bank))

    def get_leaves(self, bank: MLCBank = MLCBank.BOTH, only_moving_leaves: bool = False):
        bank = convert_to_enum(bank, MLCBank)
        leaves = copy.copy(self.moving_leaves) if only_moving_leaves else copy.copy(self._all_leaf_indices)
        if bank == MLCBank.A:
            leaves = leaves[leaves <= self.num_pairs]
        elif bank == MLCBank.B:
            leaves = leaves[leaves > self.num_pairs]
        return leaves

    def get_error_percentile(self, percentile: float = 95, bank: MLCBank = MLCBank.BOTH, only_moving_leaves: bool = False) -> float:
        leaves = self.get_leaves(bank, only_moving_leaves)
        leaves -= 1
        return np.percentile(np.abs(self.create_error_array(leaves)), percentile)

    def create_error_array(self, leaves: Sequence[int], absolute: bool = True) -> np.ndarray:
        arr = self._abs_error_all_leaves if absolute else self._error_array_all_leaves
        return arr[leaves, :]

    def create_RMS_array(self, leaves: Sequence[int]) -> np.ndarray:
        rms_array = self._RMS_array_all_leaves
        leaves -= 1          # in place, as the reference does
        if len(leaves) == 0:
            return np.array([0])
        return rms_array[leaves]

    @property
    def _abs_error_all_leaves(self) -> np.ndarray:
        return np.abs(self._error_array_all_leaves)

    @cached_property
    def _error_array_all_leaves(self) -> np.ndarray:
        err = np.zeros((self.num_leaves, self.num_snapshots))
        for leaf in range(self.num_leaves):
            err[leaf, :] = self.leaf_axes[leaf + 1].difference[self.snapshot_idx]
        return err

    def _snapshot_array(self, dtype: str = "actual") -> np.ndarray:
        if dtype not in ("actual", "expected"):
            raise ValueError(f"dtype must be 'actual' or 'expected', got {dtype!r}")
        arr = np.zeros((self.num_leaves, self.num_snapshots))
        for leaf in range(self.num_leaves):
            arr[leaf, :] = getattr(self.leaf_axes[leaf + 1], dtype)[self.snapshot_idx]
        return arr

    @cached_property
    def _RMS_array_all_leaves(self) -> np.ndarray:
        return np.array([np.sqrt(np.sum(leafdata.difference[self.snapshot_idx] ** 2) / self.num_snapshots)
                         for leafdata in self.leaf_axes.values()])

    def leaf_under_y_jaw(self, leaf_num: int) -> bool:
        """:1260-1290 (the per-leaf thickness walk, the jaw maxima over all snapshots)"""
        outer, inner, pos = 10, 5, 0
        if self.hdmlc:
            outer, inner, pos = outer / 2, inner / 2, 100
        for leaf in range(1, leaf_num + 1):
            pos += outer if (10 >= leaf or leaf >= 110) else (inner if (50 >= leaf or leaf >= 70) else outer)
        y2 = self._jaws.y2.actual.max() * 10 + 200
        y1 = 200 - self._jaws.y1.actual.max() * 10
        thickness = outer if (10 >= leaf or leaf >= 110) else (inner if (50 >= leaf or leaf >= 70) else outer)
        return pos < y1 or pos - thickness > y2

    def get_snapshot_values(self, bank_or_leaf=MLCBank.BOTH, dtype: str = "actual") -> np.ndarray:
        if isinstance(bank_or_leaf, (str, MLCBank)):
            leaves = self.get_leaves(bank=bank_or_leaf)
            leaves -= 1
        else:
            leaves = bank_or_leaf
        return self._snapshot_array(dtype)[leaves, :]


# ------------------------------------------------------------------------------------------------ subbeams (:1418-1549)
class Subbeam:
    def __init__(self, file, log_version: float):
        self.control_point = _ints(file)
        self.mu_delivered = _floats(file)
        self.rad_time = _floats(file)
        self.sequence_num = _ints(file)
        self.beam_name = _text(file, 512 if log_version >= 3 else 32, 32)

    @property
    def gantry_angle(self) -> Axis:
        return self._get_metadata_axis("gantry")

    @property
    def collimator_angle(self) -> Axis:
        return self._get_metadata_axis("collimator")

    @property
    def jaw_x1(self) -> Axis:
        return self._get_metadata_axis("jaws", "x1")

    @property
    def jaw_x2(self) -> Axis:
        return self._get_metadata_axis("jaws", "x2")

    @property
    def jaw_y1(self) -> Axis:
        return self._get_metadata_axis("jaws", "y1")

    @property
    def jaw_y2(self) -> Axis:
        return self._get_metadata_axis("jaws", "y2")

    def _get_metadata_axis(self, attr, subattr=None) -> Axis:
        ax = getattr(self._axis_data, attr)
        if subattr is not None:
            ax = getattr(ax, subattr)
        return Axis(np.median(ax.actual[self._snapshots]), np.median(ax.expected[self._snapshots]))


class SubbeamManager:
    def __init__(self, file, header):
        self.subbeams = [Subbeam(file, header.version) for _ in range(max(header.num_subbeams, 0))]

    def post_hoc_metadata(self, axis_data, source: _Source | None = None):
        for num, subbeam in enumerate(self.subbeams):
            self._set_subbeam_snapshots(axis_data, num)
            section = copy.copy(axis_data.mlc)
            section.snapshot_idx = subbeam._snapshots
            subbeam.fluence = FluenceStruct(section, axis_data.mu, axis_data.jaws, source)

    def _set_subbeam_snapshots(self, axis_data, beam_num: int):
        subbeam = self.subbeams[beam_num]
        cp = axis_data.control_point.actual
        lower = subbeam.control_point
        upper = self.subbeams[beam_num + 1].control_point if beam_num + 1 < len(self.subbeams) else cp[-1]
        keep = np.logical_and(axis_data.beam_hold.actual == 0, np.logical_and(cp >= lower, cp < upper))
        subbeam._snapshots = [i for i, b in enumerate(keep) if b]
        subbeam._axis_data = axis_data

    def __getitem__(self, item) -> Subbeam:
        return self.subbeams[item]

    def __len__(self):
        return len(self.subbeams)


# ------------------------------------------------------------------------------------------------ logs (:1552-1761)
class LogBase:
    def __init__(self, filename: str, exclude_beam_off: bool = True):
        if not is_log(filename):
            raise OSError(f"{filename} was not a valid log file")
        self.filename = filename
        self.exclude_beam_off = exclude_beam_off

    @property
    def treatment_type(self) -> str:
        """:1724-1750.  For a trajectory log the gantry spread is the std of each subbeam's median gantry angle (a scalar, so 0, or
        nan for a subbeam without snapshots); a log without subbeams raises ValueError (max() of nothing)."""
        if isinstance(self, TrajectoryLog):
            gantry_std = max(sb.gantry_angle.actual.std() for sb in self.subbeams)
            if np.isnan(gantry_std):
                return TreatmentType.IMAGING.value
        else:
            gantry_std = self.axis_data.gantry.actual.std()
        if gantry_std > 0.5:
            return TreatmentType.VMAT.value
        if self.axis_data.mu.actual.max() <= 2.1:
            return TreatmentType.IMAGING.value
        if self.axis_data.mlc.num_moving_leaves == 0 and isinstance(self, TrajectoryLog):
            return TreatmentType.STATIC_IMRT.value
        return TreatmentType.DYNAMIC_IMRT.value

    @property
    def num_beamholds(self) -> int:
        return int(np.sum(np.diff(self.axis_data.beam_hold.actual) > 0))


class DynalogHeader:  # :1764-1792
    def __init__(self, dlogdata):
        self.version = str(dlogdata[0])
        self.patient_name = dlogdata[1]
        self.plan_filename = dlogdata[2]
        self.tolerance = int(dlogdata[3][0])
        self.num_mlc_leaves = int(dlogdata[4][0]) * 2
        self.clinac_scale = int(dlogdata[5][0])


def _read_dlog_table(path):
    """-> (csv rows, snapshot data [columns, snapshots] float64) of one Dynalog file"""
    with open(path, encoding="utf-8") as f:
        rows = [line for line in csv.reader(f, delimiter=",")]
    return rows, np.array(rows[Dynalog.HEADER_LINE_LENGTH :], dtype=np.float64).transpose()


def correct_vmat_mu(mu_array: np.ndarray) -> np.ndarray:
    """:1846-1861: a VMAT Dynalog records the gantry angle in the MU column; the cumulative gantry travel normalised to 25000
    stands in for it"""
    if mu_array[-1] == 25000:
        return mu_array
    abs_diff = list(np.abs(np.diff(mu_array)))
    return np.array([0] + list(np.cumsum(abs_diff) / np.sum(abs_diff))) * 25000


class DynalogAxisData:  # :1795-1893
    def __init__(self, log, dlogdata, snapshot_data: np.ndarray | None = None, b_snapshot_data: np.ndarray | None = None):
        if snapshot_data is None:
            snapshot_data = np.array(dlogdata[6:], dtype=np.float64).transpose()
        self.num_snapshots = np.size(snapshot_data, 1)
        c = itertools.count()

        def nx():
            return snapshot_data[next(c)]

        mu = correct_vmat_mu(nx())
        self.mu = Axis(mu, mu)
        self.previous_segment_num = Axis(nx())
        self.beam_hold = Axis(nx())
        self.beam_on = Axis(nx())
        self.prior_dose_index = Axis(nx())
        self.next_dose_index = Axis(nx())
        self.gantry = GantryAxis(nx() / 10)
        self.collimator = HeadAxis(nx() / 10)
        y1, y2, x1, x2 = (HeadAxis(nx() / 10) for _ in range(4))
        self.jaws = JawStruct(x1, y1, x2, y2)
        self.carriage_A = Axis(nx() / 1000)
        self.carriage_B = Axis(nx() / 1000)
        if log.exclude_beam_off:
            snapshot_idx = np.intersect1d(np.where(self.beam_hold.actual == 0)[0], np.where(self.beam_on.actual == 1)[0])
        else:
            snapshot_idx = list(range(self.num_snapshots))
        self.mlc = MLC.from_dlog(log, self.jaws, snapshot_data, snapshot_idx, b_snapshot_data)


class Dynalog(LogBase):  # :1896-2173
    ANON_LINE = 1
    HEADER_LINE_LENGTH = 6

    def __init__(self, filename, exclude_beam_off: bool = True):
        super().__init__(filename, exclude_beam_off)
        if not is_dlog(self.filename):
            raise NotADynalogError(f"{self.filename} was not a valid Dynalog file")
        if not self._has_other_file:
            raise DynalogMatchError("Didn't find the matching dynalog file")
        dlgdata, a_table = _read_dlog_table(self.a_logfile)
        self.header = DynalogHeader(dlgdata)
        self.axis_data = DynalogAxisData(self, dlgdata, a_table)
        self.fluence = FluenceStruct(self.axis_data.mlc, self.axis_data.mu, self.axis_data.jaws)

    def snapshot_idx(self, axis_data):
        if self.exclude_beam_off:
            return np.intersect1d(np.where(axis_data.beam_hold.actual == 0)[0], np.where(axis_data.beam_on.actual == 1)[0])
        return list(range(self.num_snapshots))

    @property
    def _has_other_file(self) -> bool:
        return self.identify_other_file(self.filename, raise_find_error=False) is not None

    @cached_property
    def a_logfile(self) -> str:
        other = self.identify_other_file(self.filename)
        return self.filename if osp.basename(self.filename).startswith("A") else other

    @cached_property
    def b_logfile(self) -> str:
        other = self.identify_other_file(self.filename)
        return self.filename if osp.basename(self.filename).startswith("B") else other

    @staticmethod
    def identify_other_file(first_dlg_file: str, raise_find_error: bool = True) -> str:
        dlg_dir, dlg_file = osp.split(first_dlg_file)
        if dlg_file.startswith("A"):
            file2get = dlg_file.replace("A", "B", 1)
        elif dlg_file.startswith("B"):
            file2get = dlg_file.replace("B", "A", 1)
        else:
            raise ValueError("Unable to decipher log names; ensure dynalogs start with 'A' and 'B'")
        other = osp.join(dlg_dir, file2get)
        if osp.isfile(other):
            return other
        if raise_find_error:
            raise FileNotFoundError("Complementary dlg file not found; ensure A and B-file are in same directory.")


class TrajectoryLogHeader:  # :2258-2313
    def __init__(self, file):
        f = file
        self.header = _text(f, 16)
        self.version = float(_text(f, 16))
        self.header_size = _ints(f)
        self.sampling_interval = _ints(f)
        self.num_axes = _ints(f)
        self.axis_enum = _ints(f, self.num_axes)
        self.samples_per_axis = _ints(f, self.num_axes)
        self.num_mlc_leaves = self.samples_per_axis[-1] - 2
        self.axis_scale = _ints(f)
        self.num_subbeams = _ints(f)
        self.is_truncated = _ints(f)
        self.num_snapshots = _ints(f)
        self.mlc_model = _ints(f)
        if self.version >= 4.0:
            self.metadata = Metadata(f, self.num_axes)
        else:
            f.seek(1024 - (64 + self.num_axes * 8), 1)


class Metadata:
    """Trajectory-log v4.0 metadata (:2316-2336): 745 bytes of "name\\tvalue" lines.  The reserved section that follows is NOT the
    size the file specification gives: it is shortened by the metadata, 1024 - (64 + num_axes * 8) - 745 bytes."""

    def __init__(self, stream, num_axes: int):
        fields = _text(stream, 745, 1024 - (64 + num_axes * 8) - 745).split("\r\n")
        self.patient_id: str = fields[0].split("\t")[1]
        self.plan_name: str = fields[1].split("\t")[1]
        self.sop_instance_uid: str = fields[2].split("\t")[1]
        self.mu_planned: float = float(fields[3].split("\t")[1])
        self.mu_remaining: float = float(fields[4].split("\t")[1])
        self.energy: str = fields[5].split("\t")[1]
        self.beam_name: str = fields[6].split("\t")[1]


def _get_axis(snapshot_data, column, axis_type):  # :2913-2931
    return axis_type(expected=snapshot_data[:, column], actual=snapshot_data[:, column + 1])


class TrajectoryLogAxisData:  # :2176-2255
    def __init__(self, log, snapshot_data: np.ndarray, subbeams):
        clm = itertools.count(step=2)
        self.collimator = _get_axis(snapshot_data, next(clm), HeadAxis)
        self.gantry = _get_axis(snapshot_data, next(clm), GantryAxis)
        y1 = _get_axis(snapshot_data, next(clm), HeadAxis)
        y2 = _get_axis(snapshot_data, next(clm), HeadAxis)
        x1 = _get_axis(snapshot_data, next(clm), HeadAxis)
        x2 = _get_axis(snapshot_data, next(clm), HeadAxis)
        self.jaws = JawStruct(x1, y1, x2, y2)
        vrt, lng, lat, rtn = (_get_axis(snapshot_data, next(clm), CouchAxis) for _ in range(4))
        if log.header.version >= 3:
            pitch = _get_axis(snapshot_data, next(clm), CouchAxis)
            roll = _get_axis(snapshot_data, next(clm), CouchAxis)
        else:
            pitch = roll = None
        self.couch = CouchStruct(vrt, lng, lat, rtn, pitch, roll)
        self.mu = _get_axis(snapshot_data, next(clm), BeamAxis)
        self.beam_hold = _get_axis(snapshot_data, next(clm), BeamAxis)
        self.control_point = _get_axis(snapshot_data, next(clm), BeamAxis)
        self.carriage_A = _get_axis(snapshot_data, next(clm), HeadAxis)
        self.carriage_B = _get_axis(snapshot_data, next(clm), HeadAxis)
        if log.exclude_beam_off:
            snapshot_idx = np.where(self.beam_hold.actual == 0)[0]
        else:
            snapshot_idx = list(range(log.header.num_snapshots))
        self.mlc = MLC.from_tlog(log, subbeams, self.jaws, snapshot_data, snapshot_idx, clm)


def _tlog_source(log: "TrajectoryLog", body: np.ndarray) -> _Source:
    """column table of a trajectory log's raw float32 body: (expected, actual) per sample"""
    n_single = 15 if log.header.version >= 3 else 13
    mu = 2 * (n_single - 3)
    leaf1 = 2 * (n_single + 2)
    return _Source(body, (mu + 1, mu), 2 * 4 + 1, 2 * 5 + 1, (leaf1 + 1, leaf1))


class TrajectoryLog(LogBase):  # :2339-2743
    ANON_LINE = 0

    def __init__(self, filename: str, exclude_beam_off: bool = True, *, _body: np.ndarray | None = None):
        super().__init__(filename, exclude_beam_off)
        self._read_txt_file()
        with open(self.filename, mode="rb") as f:
            self.header = TrajectoryLogHeader(f)
            self.subbeams = SubbeamManager(f, self.header)
            self._body_offset = f.tell()
            count = sum(self.header.samples_per_axis) * 2 * self.header.num_snapshots
            if _body is None:
                _body = np.empty(max(count, 0), np.float32)
                got = f.readinto(memoryview(_body).cast("B")) or 0
                if got != 4 * count:
                    raise struct.error(f"unpack requires a buffer of {4 * count} bytes")
        body = _body.reshape(self.header.num_snapshots, -1)
        # decode_binary(f, float, n): the float32 values widened to float64 (:2211-2215)
        self.axis_data = TrajectoryLogAxisData(self, np.asarray(body).astype(np.float64), self.subbeams)
        self._source = _tlog_source(self, body)
        self.subbeams.post_hoc_metadata(self.axis_data, self._source)
        if not self.treatment_type == TreatmentType.IMAGING.value:
            self.fluence = FluenceStruct(self.axis_data.mlc, self.axis_data.mu, self.axis_data.jaws, self._source)

    @property
    def txt_filename(self) -> str | None:
        if self.txt is not None:
            return self.filename.replace(".bin", ".txt")

    def _read_txt_file(self) -> None:
        self.txt = None
        if ".bin" in str(self.filename):
            txt_filename = str(self.filename).replace(".bin", ".txt")
            if osp.isfile(txt_filename):
                self.txt = {}
                with open(txt_filename, encoding="utf-8") as f:
                    for line in f.readlines():
                        items = line.split(":")
                        if len(items) == 2:
                            self.txt[items[0].strip()] = items[1].strip()

    @property
    def is_hdmlc(self) -> bool:
        return self.header.mlc_model == 3


# ------------------------------------------------------------------------------------------------ files (:2800-2910)
def is_log(filename) -> bool:
    return is_tlog(filename) or is_dlog(filename)


def is_tlog(filename) -> bool:
    return _is_log(filename, ("VOSTL",))


def is_dlog(filename) -> bool:
    return _is_log(filename, ("B", "A"))


def _is_log(filename, keys: Sequence[str]) -> bool:
    if osp.isfile(filename):
        try:
            with open(filename, mode="rb") as f:
                sample = f.read(5).decode()
            return any(k in sample for k in keys)
        except Exception:
            return False
    return False


def load_log(file_or_dir: str, exclude_beam_off: bool = True, recursive: bool = True):
    """A TrajectoryLog or Dynalog for a file, MachineLogs for a directory or a ZIP archive (a ZIP of one log: that log)."""
    if osp.isfile(file_or_dir):
        if zipfile.is_zipfile(file_or_dir):
            logs = MachineLogs.from_zip(file_or_dir)
            return logs[0] if len(logs) == 1 else logs
        if not is_log(file_or_dir):
            raise NotALogError("Not a valid log")
        if is_tlog(file_or_dir):
            return TrajectoryLog(file_or_dir, exclude_beam_off)
        return Dynalog(file_or_dir, exclude_beam_off)
    if osp.isdir(file_or_dir):
        return MachineLogs(file_or_dir, recursive)
    raise NotALogError(f"'{file_or_dir}' did not point to a valid file, directory, or ZIP archive")


def _retrieve_filenames(directory, func, recursive: bool = True) -> list[str]:  # core/io.py:119-152
    out = []
    for pdir, _, files in os.walk(directory):
        for file in files:
            fn = osp.join(pdir, file)
            if func(fn):
                out.append(fn)
        if not recursive:
            break
    return out


def _get_log_filenames(directory: str, recursive: bool = True) -> list:
    tlogs = _retrieve_filenames(directory, is_tlog, recursive)
    dlogs = _retrieve_filenames(directory, is_dlog, recursive)
    idx = 0
    while idx < len(dlogs):        # keep one file of every A / B pair; drop a Dynalog without its companion
        opp = Dynalog.identify_other_file(dlogs[idx], raise_find_error=False)
        if opp in dlogs:
            del dlogs[dlogs.index(opp)]
        else:
            del dlogs[idx]
            idx -= 1
        idx += 1
    return tlogs + dlogs


# ------------------------------------------------------------------------------------------------ batches
@dataclass
class LogResult:
    """One log of analyze_batch: the figures report_basic_parameters prints (:1694-1722).  Statistics are None for an imaging
    field (the reference computes none); the map-level objects stay reachable through ``log``."""

    path: str
    treatment_type: str
    rms_avg: float | None
    rms_max: float | None
    error_p95: float | None
    num_beamholds: int
    avg_gamma: float | None
    pass_prcnt: float | None
    log: object


def _gamma_batch(logs, doseTA, distTA, threshold, resolution, equal_aspect: bool = False, pinned: bool = True,
                 keep_maps: bool = True) -> None:
    """GammaFluence.calc_map(doseTA, distTA, threshold, resolution) of every log with a fluence, batched: fluences of one map
    shape in one epid_log_fluence launch per chunk (at most about 2 GB per map batch), then one device gamma pipeline per chunk.
    Only two numbers per log come back to the host.  keep_maps: every log keeps its actual, expected and gamma maps on the device
    (3 x 8 x rows x columns bytes per log, e.g. 5.8 MB at 0.1 mm, 384 MB with equal_aspect); otherwise each chunk's maps are freed
    once its numbers are back and only the gamma scalars (avg_gamma, pass_prcnt, doseTA, distTA, threshold) are set."""
    todo = [lg for lg in logs if hasattr(lg, "fluence")]
    fresh = [lg for lg in todo if not (lg.fluence.actual.is_map_calced() or lg.fluence.expected.is_map_calced())]
    for lg in todo:
        if lg not in fresh:                       # a map the caller computed before: the reference's per-log path reuses it
            lg.fluence.gamma.calc_map(doseTA, distTA, threshold, resolution)
    groups: dict[int, list] = {}
    for lg in fresh:
        groups.setdefault(_fluence_rows(lg.fluence.actual, resolution, equal_aspect), []).append(lg)
    ctx = nat.Context.default()
    W = int(MLC_FOV_WIDTH_MM / resolution)
    for R, members in groups.items():
        chunk = max(1, int(2e9 // (8 * R * W)))
        for c0 in range(0, len(members), chunk):
            part = members[c0 : c0 + chunk]
            a, e = _compute_fluences([(lg.fluence, lg.fluence.actual._src()) for lg in part], resolution, equal_aspect, 3, pinned, ctx)
            g, avg, pct = _gamma_maps(a.batch, e.batch, doseTA, distTA, threshold, resolution, ctx)
            if not keep_maps:
                for b in (a.batch, e.batch, g):
                    b.free()
                for i, lg in enumerate(part):
                    gf = lg.fluence.gamma
                    gf.avg_gamma, gf.pass_prcnt = avg[i], pct[i]
                    gf.distTA, gf.doseTA, gf.threshold = distTA, doseTA, threshold
                continue
            gm = _Maps(g)
            key = (resolution, equal_aspect)
            for i, lg in enumerate(part):
                lg.fluence.actual._set(a, i, resolution, key)
                lg.fluence.expected._set(e, i, resolution, key)
                lg.fluence.gamma._finish(gm, i, avg[i], pct[i], doseTA, distTA, threshold, resolution)


def _read_all(paths, exclude_beam_off: bool, threads: int = 8):
    """Every log of `paths`: trajectory-log bodies `readinto` their 16-byte-aligned slots of ONE page-locked arena, Dynalogs parsed
    on the host and their fp64 column tables copied into the same arena."""
    from concurrent.futures import ThreadPoolExecutor

    metas = []
    for p in paths:
        p = str(p)
        if not is_log(p):
            raise NotALogError("Not a valid log")
        if is_tlog(p):
            with open(p, "rb") as f:
                hd = TrajectoryLogHeader(f)
                SubbeamManager(f, hd)
                off = f.tell()
            count = sum(hd.samples_per_axis) * 2 * hd.num_snapshots
            metas.append(("t", p, off, 4 * max(count, 0)))
        else:
            metas.append(("d", p, 0, 0))
    with ThreadPoolExecutor(max(1, min(threads, len(metas)))) as pool:
        dlogs = dict(zip([m[1] for m in metas if m[0] == "d"],
                         pool.map(lambda p: Dynalog(p, exclude_beam_off), [m[1] for m in metas if m[0] == "d"])))
        srcs = {p: lg.fluence.actual._src() for p, lg in dlogs.items()}
        sizes = [m[3] if m[0] == "t" else srcs[m[1]].buf.nbytes for m in metas]
        offs = np.concatenate([[0], np.cumsum([_slot(s) for s in sizes])]).astype(np.int64)
        arena = nat.pinned_empty((max(int(offs[-1]), 16),), np.uint8)

        def fill(i):
            kind, p, off, nbytes = metas[i]
            o = int(offs[i])
            if kind == "d":
                buf = srcs[p].buf
                arena[o : o + buf.nbytes] = buf.reshape(-1).view(np.uint8)
                return None
            with open(p, "rb", buffering=0) as f:
                f.seek(off)
                mv = memoryview(arena[o : o + nbytes])
                got = 0
                while got < nbytes:
                    r = f.readinto(mv[got:])
                    if not r:
                        raise struct.error(f"unpack requires a buffer of {nbytes} bytes")
                    got += r
            return None

        list(pool.map(fill, range(len(metas))))
        logs = []
        for i, (kind, p, off, nbytes) in enumerate(metas):
            o = int(offs[i])
            if kind == "d":
                lg = dlogs[p]
                buf = srcs[p].buf
                view = _ArenaView(arena, o, buf.shape, np.float64)
                lg.fluence.actual._source = lg.fluence.expected._source = _Source(view, srcs[p].col_mu, srcs[p].col_x1, srcs[p].col_x2,
                                                                                  srcs[p].col_leaf)
            else:
                lg = TrajectoryLog(p, exclude_beam_off, _body=_ArenaView(arena, o, (nbytes // 4,), np.float32))
            logs.append(lg)
    return logs


def _ArenaView(arena: np.ndarray, off: int, shape, dtype) -> np.ndarray:
    """a typed view of arena[off:] that remembers its arena (so one launch uses the arena in place)"""
    v = _Viewed(arena[off : off + int(np.prod(shape)) * np.dtype(dtype).itemsize].view(dtype).reshape(shape))
    v._arena = arena
    return v


class _Viewed(np.ndarray):
    """ndarray subclass that carries the arena it views; reshape / views keep it"""

    def __new__(cls, a):
        return np.asarray(a).view(cls)

    def __array_finalize__(self, obj):
        self._arena = getattr(obj, "_arena", None)


def analyze_batch(paths, resolution: float = 0.1, doseTA: float = 1, distTA: float = 1, threshold: float = 0.1,
                  equal_aspect: bool = False, exclude_beam_off: bool = True, keep_maps: bool = False) -> list[LogResult]:
    """Load every log of `paths` (trajectory logs and Dynalogs, in any mix and with any snapshot counts) and compute, per log, what
    ``report_basic_parameters`` reports: RMS average / maximum and the 95th-percentile leaf error (host, the reference's numpy),
    the number of beam holds and the fluence gamma (``GammaFluence.calc_map(doseTA, distTA, threshold, resolution)`` on fluences
    computed with ``calc_map(resolution, equal_aspect)``), on the GPU in one launch sequence per map shape and chunk.  By default
    the maps are freed once each chunk's numbers are back, so device memory stays bounded by one chunk whatever the number of logs;
    keep_maps=True keeps every log's actual, expected and gamma maps on the device (nothing is downloaded until a log's
    ``.fluence.*.array`` is read) at 3 x 8 x rows x columns bytes per log."""
    logs = _read_all(paths, exclude_beam_off)
    _gamma_batch(logs, doseTA, distTA, threshold, resolution, equal_aspect, keep_maps=keep_maps)
    out = []
    for p, lg in zip(paths, logs):
        tt = lg.treatment_type
        if tt == TreatmentType.IMAGING.value or not hasattr(lg, "fluence"):
            out.append(LogResult(str(p), tt, None, None, None, lg.num_beamholds, None, None, lg))
            continue
        mlc = lg.axis_data.mlc
        out.append(LogResult(str(p), tt, mlc.get_RMS_avg(only_moving_leaves=False), mlc.get_RMS_max(),
                             mlc.get_error_percentile(95, only_moving_leaves=False), lg.num_beamholds, lg.fluence.gamma.avg_gamma,
                             lg.fluence.gamma.pass_prcnt, lg))
    return out


class MachineLogs(list):  # :84-312
    """The logs of a directory (a list); ``avg_gamma`` / ``avg_gamma_pct`` compute every log's fluence gamma in one batch.  As in
    the reference every log keeps its maps afterwards, here on the device: 3 x 8 x 60 x int(400 / resolution) bytes per log."""

    def __init__(self, folder: str, recursive: bool = True):
        super().__init__()
        self.load_folder(folder, recursive)

    @classmethod
    def from_zip(cls, zfile: str):
        with tempfile.TemporaryDirectory() as tmp:
            with zipfile.ZipFile(zfile) as z:
                z.extractall(tmp)
            return cls(tmp)

    @property
    def num_logs(self) -> int:
        return len(self)

    @property
    def num_tlogs(self) -> int:
        return sum(isinstance(lg, TrajectoryLog) for lg in self)

    @property
    def num_dlogs(self) -> int:
        return sum(isinstance(lg, Dynalog) for lg in self)

    def load_folder(self, directory: str, recursive: bool = True):
        files = _get_log_filenames(directory, recursive=recursive)
        if len(files) == 0:
            print("No logs found.")
            return
        print(f"{len(files)} logs found.")
        for idx, file in enumerate(files):
            self.append(file)
            print(f"Log loaded: {idx + 1} of {len(files)}", end="\r")
        print("")

    def _check_empty(self) -> None:
        if len(self) == 0:
            raise ValueError("No logs have been loaded yet.")

    def append(self, obj, recursive: bool = True) -> None:
        if isinstance(obj, str):
            if is_log(obj):
                super().append(load_log(obj))
            elif osp.isdir(obj):
                for file in _retrieve_filenames(obj, lambda x: True):
                    self.append(file)
        elif isinstance(obj, (Dynalog, TrajectoryLog)):
            super().append(obj)
        else:
            raise TypeError("Can only append MachineLog or string pointing to a log or log directory.")

    def _gammas(self, doseTA, distTA, threshold, resolution):
        self._check_empty()
        for lg in self:
            if not hasattr(lg, "fluence"):
                lg.fluence               # noqa: B018 -- the reference's AttributeError for an imaging trajectory log
        _gamma_batch(list(self), doseTA, distTA, threshold, resolution)
        return [lg.fluence.gamma for lg in self]

    def avg_gamma(self, doseTA: float = 1, distTA: float = 1, threshold: float = 0.1, resolution: float = 0.1) -> float:
        gammas = self._gammas(doseTA, distTA, threshold, resolution)
        return np.array([g.avg_gamma for g in gammas], dtype=np.float64).mean()

    def avg_gamma_pct(self, doseTA: float = 1, distTA: float = 1, threshold: float = 0.1, resolution: float = 0.1) -> float:
        gammas = self._gammas(doseTA, distTA, threshold, resolution)
        return np.array([g.pass_prcnt for g in gammas], dtype=np.float64).mean()
