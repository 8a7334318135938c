"""``pylinac.core.gamma.gamma_2d`` (reference core/gamma.py:229-330; Low et al. 2004, Table I) on the GPU, for one pair of images
or a batch of pairs.  Every map is bit-identical to the reference's: the search over the disk, the normalisation and numpy 2's dtype
promotion run in ``csrc/gamma2d.cu``; the host builds the disk of offsets and checks the arguments.
"""
from __future__ import annotations

import numpy as np

from .. import _native as nat

# numpy inputs go to the device in chunks of at most this many reference + evaluation pixels
_CHUNK_PIXELS = 1 << 26


def _disk_offsets(distance_to_agreement: int) -> tuple[np.ndarray, np.ndarray]:
    """Offsets of skimage.draw.disk((0, 0), dta + 1) as (int32 [k, 2], dist_r_2 float64 [k]), sorted by dist_r_2 with raster order
    breaking ties.  The membership test is skimage's floating-point ``(r / R)**2 + (c / R)**2 < 1`` over its float grid, not the
    integer r**2 + c**2 < R**2: at R = 41 it keeps (+-40, +-9) and (+-9, +-40), which lie on the circle.  dist_r_2 is the
    reference's ``(rr / dta)**2 + (cc / dta)**2`` (nan for dta = 0, as in the reference)."""
    radius = distance_to_agreement + 1
    grid = np.arange(2 * radius + 1, dtype=np.float64) - radius
    rr, cc = np.nonzero((grid[:, None] / radius) ** 2 + (grid[None, :] / radius) ** 2 < 1)
    rr, cc = rr - radius, cc - radius
    with np.errstate(divide="ignore", invalid="ignore"):
        dist2 = (rr / distance_to_agreement) ** 2 + (cc / distance_to_agreement) ** 2
    order = np.argsort(dist2, kind="stable")
    return np.stack([rr[order], cc[order]], axis=1).astype(np.int32), dist2[order]


def _shape_text(shape) -> str:
    return "(" + ",".join(str(s) for s in shape) + ")"


def _check(ref_shape, eval_shape, distance_to_agreement, global_dose) -> None:
    """The reference's exceptions for the frame shapes [h, w] and the distance, in the order it meets them."""
    if not global_dose and eval_shape != ref_shape:
        try:
            np.broadcast_shapes(eval_shape, ref_shape)
        except ValueError:
            raise ValueError(f"operands could not be broadcast together with shapes {_shape_text(eval_shape)} "
                             f"{_shape_text(ref_shape)} ") from None
        raise ValueError(f"local dose needs a reference and an evaluation of one shape, got {ref_shape} and {eval_shape}")
    if isinstance(distance_to_agreement, (bool, np.bool_)) or not isinstance(distance_to_agreement, (int, np.integer)):
        raise TypeError("`pad_width` must be of integral type.")
    if distance_to_agreement < 0:
        raise ValueError("index can't contain negative values")
    if global_dose and (eval_shape[0] < ref_shape[0] or eval_shape[1] < ref_shape[1]):
        # the reference raises IndexError only once a pixel above the threshold reaches past the evaluation
        raise ValueError(f"the evaluation {eval_shape} is smaller than the reference {ref_shape}")


def _stats(ctx: nat.Context, maps: nat.Batch) -> dict:
    s, cnt, passing = nat.gamma_stats(ctx, maps)
    with np.errstate(invalid="ignore", divide="ignore"):
        return {"mean": s / cnt, "evaluated": cnt, "pass_rate": passing / cnt * 100}


def gamma_2d(
    reference: np.ndarray,
    evaluation: np.ndarray,
    dose_to_agreement: float = 1,
    distance_to_agreement: int = 1,
    gamma_cap_value: float = 2,
    global_dose: bool = True,
    dose_threshold: float = 5,
    fill_value: float = np.nan,
) -> np.ndarray:
    """Compute a 2D gamma of two 2D numpy arrays (reference core/gamma.py:229-330), bit-identical to the reference.

    The distance to agreement is in elements.  Doses are normalised by ``dose_to_agreement`` percent of the reference's maximum
    (``global_dose``) or of the reference pixel itself; reference pixels whose normalised value is nan or below
    ``dose_threshold / 100`` take ``fill_value``; the others take the minimum over the disk of radius DTA around them of the
    squared normalised distance plus squared normalised dose difference, square-rooted and capped at ``gamma_cap_value``.  The
    evaluation is edge-padded, so in global mode it may be larger than the reference.

    Divergence from the reference: an evaluation smaller than the reference raises ``ValueError`` up front (the reference raises
    ``IndexError`` only when a pixel above the threshold reaches past it).
    """
    if reference.ndim != 2 or evaluation.ndim != 2:
        raise ValueError(
            f"Reference and evaluation arrays must be 2D. Got reference: {reference.ndim} and evaluation: {evaluation.ndim}"
        )
    return gamma_2d_batch(reference[None], evaluation[None], dose_to_agreement, distance_to_agreement, gamma_cap_value,
                          global_dose, dose_threshold, fill_value)[0]


def gamma_2d_batch(
    references,
    evaluations,
    dose_to_agreement: float = 1,
    distance_to_agreement: int = 1,
    gamma_cap_value: float = 2,
    global_dose: bool = True,
    dose_threshold: float = 5,
    fill_value: float = np.nan,
    *,
    stats: bool = False,
    device: bool = False,
    full_search: bool = False,
    ctx: nat.Context | None = None,
):
    """``gamma_2d`` of n pairs: ``references`` [n, h, w] and ``evaluations`` [n, he, we], numpy arrays or device batches
    (``_native.Batch``).  Returns the float64 maps [n, h, w] as numpy, or as a device batch with ``device=True``.

    numpy inputs go through in chunks of pairs (one upload, launch sequence and download each); device batches, and numpy inputs with
    ``device=True``, in one launch sequence.

    ``stats=True`` also returns ``{"mean", "evaluated", "pass_rate"}``, arrays [n]: the mean of the non-nan values, their count and
    count(gamma < 1) / evaluated * 100 (the log analyzer's pass percent; nan where nothing was evaluated).  With a ``fill_value`` that
    is not nan, the pixels below the threshold count as evaluated values.

    ``full_search=True`` visits every offset of the disk instead of stopping once no later offset can lower the minimum; the maps are
    identical either way.
    """
    on_device = isinstance(references, nat.Batch), isinstance(evaluations, nat.Batch)
    if on_device[0]:
        (n, h, w), _ = references.shape_dtype
    else:
        references = np.asarray(references)
        if references.ndim != 3:
            raise ValueError(f"references must be [n, h, w], got {references.ndim} dimensions")
        n, h, w = references.shape
    if on_device[1]:
        (ne, he, we), _ = evaluations.shape_dtype
    else:
        evaluations = np.asarray(evaluations)
        if evaluations.ndim != 3:
            raise ValueError(f"evaluations must be [n, h, w], got {evaluations.ndim} dimensions")
        ne, he, we = evaluations.shape
    if n != ne:
        raise ValueError(f"{n} references but {ne} evaluations")
    _check((h, w), (he, we), distance_to_agreement, global_dose)
    if n == 0 or h * w == 0:
        if global_dose and h * w == 0:
            np.empty((0,)).max()                    # the reference's ndarray.max() of an empty array
        np.pad(np.empty((h, w)), int(distance_to_agreement), mode="edge")     # and np.pad's error for an empty frame
        out = np.empty((n, h, w))
        empty = {"mean": np.full(n, np.nan), "evaluated": np.zeros(n, np.int64), "pass_rate": np.full(n, np.nan)}
        return (out, empty) if stats else out

    offsets, dist2 = _disk_offsets(int(distance_to_agreement))
    args = (dose_to_agreement / 100, dose_threshold / 100, float(gamma_cap_value), float(gamma_cap_value ** 2), float(fill_value),
            bool(global_dose), offsets, dist2, full_search)
    ctx = ctx or nat.Context.default()
    if device or any(on_device):
        with nat.batch_for(ctx, references) as rb, nat.batch_for(ctx, evaluations) as eb:
            maps = nat.gamma2d(ctx, rb, eb, *args)
        result = maps if device else maps.download()
        if not stats:
            return result
        st = _stats(ctx, maps)
        if not device:
            maps.free()
        return result, st

    out = np.empty((n, h, w))
    st = {"mean": np.empty(n), "evaluated": np.empty(n, np.int64), "pass_rate": np.empty(n)}
    step = max(1, _CHUNK_PIXELS // (h * w + he * we))
    for i in range(0, n, step):
        with nat.Batch.upload(ctx, references[i:i + step]) as rb, nat.Batch.upload(ctx, evaluations[i:i + step]) as eb, \
                nat.gamma2d(ctx, rb, eb, *args) as maps:
            out[i:i + step] = maps.download()
            if stats:
                for key, v in _stats(ctx, maps).items():
                    st[key][i:i + step] = v
    return (out, st) if stats else out


# ------------------------------------------------------------------------------------------------------- gamma_geometric / gamma_1d
def _not_1d(reference, evaluation) -> bool:
    return reference.ndim != 1 or evaluation.ndim != 1


def _ndim_error(reference, evaluation) -> ValueError:
    return ValueError(
        f"Reference and evaluation arrays must be 1D. Got reference: {reference.ndim} and evaluation: {evaluation.ndim}"
    )


def _is_monotonic(array: np.ndarray) -> bool:
    """array_utils.is_monotonic with its validators (reference core/array_utils.py:422-436)"""
    if not array.size:
        raise ValueError("Array must not be empty")
    if array.ndim > 1:
        raise ValueError(f"Array was multidimensional. Must pass 1D array; found {array.ndim}")
    d = np.diff(array)
    return bool(np.all(d > 0) or np.all(d < 0))


def _float64_coordinates(*arrays) -> None:
    for a in arrays:
        if a.dtype != np.float64:
            raise TypeError(f"coordinates must be float64 or integer so that the window search and the sample positions run in "
                            f"float64, got {a.dtype}")


def _rows(arrays) -> list[np.ndarray]:
    return [np.asarray(a) for a in arrays]


def _coordinate_rows(coordinates, n: int) -> list:
    if coordinates is None:
        return [None] * n
    rows = [None if c is None else np.asarray(c) for c in coordinates]
    if len(rows) != n:
        raise ValueError(f"{n} pairs but {len(rows)} coordinate arrays")
    return rows


def _offsets(lengths) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(lengths, dtype=np.int64)]).astype(np.int64)


def _assign(out: np.ndarray, mask: np.ndarray, values: np.ndarray) -> np.ndarray:
    """``out[i] = v`` at the evaluated points as the reference assigns them: into an integer array (an integer ``fill_value``) a float
    is truncated, and a nan or an infinity raises Python's error."""
    if out.dtype.kind != "f" and not np.isfinite(values).all():
        for i, v in zip(np.flatnonzero(mask), values):
            out[i] = v
    out[mask] = values
    return out


def gamma_geometric(
    reference: np.ndarray,
    evaluation: np.ndarray,
    reference_coordinates: np.ndarray | None = None,
    evaluation_coordinates: np.ndarray | None = None,
    dose_to_agreement: float = 1,
    distance_to_agreement: float = 1,
    gamma_cap_value: float = 2,
    dose_threshold: float = 5,
    fill_value: float = np.nan,
) -> np.ndarray:
    """Ju et al. geometric gamma of two 1-D profiles (reference core/gamma.py:105-226), bit-identical to the reference; a batch of one
    for ``gamma_geometric_batch``.

    ``dose_to_agreement`` is in % of the reference's maximum, ``distance_to_agreement`` in the units of the coordinates (element
    indices when they are None).  Each reference point at or above ``dose_threshold`` (in units of the dose criterion) takes the
    least distance, in the normalised (x / DTA, dose / dose criterion) plane, to the evaluation's segments in a window around it,
    capped at ``gamma_cap_value``; the others take ``fill_value``, in an array ``np.full(len(reference), fill_value)``.

    As in the reference, the window is found by subtracting the unnormalised ``distance_to_agreement`` from the normalised x: it
    spans +-DTA in normalised units, i.e. +-DTA**2 in the caller's units, widened by one sample each side.  A nan that reaches a
    segment raises ``numpy.linalg.LinAlgError`` as the reference's ``pinv`` does.

    Divergence from the reference: float32 (or other non-float64 floating) coordinates raise ``TypeError``; the reference runs the
    window search in float32 for them.
    """
    if _not_1d(reference, evaluation):
        raise _ndim_error(reference, evaluation)
    return gamma_geometric_batch([reference], [evaluation], None if reference_coordinates is None else [reference_coordinates],
                                 None if evaluation_coordinates is None else [evaluation_coordinates], dose_to_agreement,
                                 distance_to_agreement, gamma_cap_value, dose_threshold, fill_value)[0]


def _prepare_geometric(reference, evaluation, rc, ec, dose_to_agreement, distance_to_agreement, dose_threshold):
    """the reference's checks and O(n) preparation (core/gamma.py:147-187), in its expressions so that numpy's promotion applies"""
    if _not_1d(reference, evaluation):
        raise _ndim_error(reference, evaluation)
    if distance_to_agreement <= 0:
        raise ValueError("Dose to agreement must be greater than 0")       # the reference's messages, swapped as it has them
    if dose_to_agreement <= 0:
        raise ValueError("Distance to agreement must be greater than 0")
    if rc is None:
        rc = np.arange(len(reference), dtype=float)
    if not _is_monotonic(rc):
        raise ValueError("Reference x-values must be monotonically increasing or decreasing")
    if len(reference) != len(rc):
        raise ValueError(f"Reference and reference_x_values must be the same length. Got reference: {len(reference)} and "
                         f"reference_x_values: {len(rc)}")
    if ec is None:
        ec = np.arange(len(evaluation), dtype=float)
    if not _is_monotonic(ec):
        raise ValueError("Evaluation x-values must be monotonically increasing or decreasing")
    if len(evaluation) != len(ec):
        raise ValueError(f"Evaluation and evaluation_x_values must be the same length. Got evaluation: {len(evaluation)} and "
                         f"evaluation_x_values: {len(ec)}")
    threshold = float(dose_threshold) / float(dose_to_agreement)
    norm_ref = reference.astype(float) * 100 / (reference.max() * dose_to_agreement)
    norm_eval = evaluation.astype(float) * 100 / (reference.max() * dose_to_agreement)
    norm_ref_x = rc / distance_to_agreement
    norm_eval_x = ec / distance_to_agreement
    _float64_coordinates(norm_ref_x, norm_eval_x)
    mask = ~(norm_ref < threshold)
    if mask.any() and len(evaluation) < 2:
        raise ValueError("min() iterable argument is empty")    # no segment in the window
    decreasing = bool(np.all(np.diff(norm_eval_x) < 0))
    return mask, norm_eval_x, np.asarray(norm_eval, dtype=np.float64), decreasing, norm_ref_x[mask], norm_ref[mask]


def gamma_geometric_batch(
    references,
    evaluations,
    reference_coordinates=None,
    evaluation_coordinates=None,
    dose_to_agreement: float = 1,
    distance_to_agreement: float = 1,
    gamma_cap_value: float = 2,
    dose_threshold: float = 5,
    fill_value: float = np.nan,
    *,
    ctx: nat.Context | None = None,
) -> list[np.ndarray]:
    """``gamma_geometric`` of n pairs of 1-D profiles, whose lengths may differ from pair to pair: ``references`` and ``evaluations``
    are sequences of n arrays (a 2-D array is a sequence of rows), the coordinates None or one array (or None) per pair.  Returns
    the list of the n gamma arrays.  Every pair's arguments are checked, with the reference's exceptions, before one device call
    (one upload, one kernel, one download) computes them all."""
    refs, evs = _rows(references), _rows(evaluations)
    if len(refs) != len(evs):
        raise ValueError(f"{len(refs)} references but {len(evs)} evaluations")
    n = len(refs)
    rcs, ecs = _coordinate_rows(reference_coordinates, n), _coordinate_rows(evaluation_coordinates, n)
    preps = [_prepare_geometric(refs[i], evs[i], rcs[i], ecs[i], dose_to_agreement, distance_to_agreement, dose_threshold)
             for i in range(n)]
    if n == 0:
        return []
    ctx = ctx or nat.Context.default()
    g, fail = nat.gamma_geometric(
        ctx, _offsets([len(p[1]) for p in preps]), _offsets([len(p[4]) for p in preps]), [p[3] for p in preps],
        np.concatenate([p[1] for p in preps]), np.concatenate([p[2] for p in preps]), np.concatenate([p[4] for p in preps]),
        np.concatenate([p[5] for p in preps]), float(distance_to_agreement), float(gamma_cap_value))
    if fail.any():
        raise np.linalg.LinAlgError("SVD did not converge")
    out, at = [], 0
    for ref, p in zip(refs, preps):
        k = len(p[4])
        out.append(_assign(np.full(len(ref), fill_value), p[0], g[at:at + k]))
        at += k
    return out


def gamma_1d(
    reference: np.ndarray,
    evaluation: np.ndarray,
    reference_coordinates: np.ndarray | None = None,
    evaluation_coordinates: np.ndarray | None = None,
    dose_to_agreement: float = 1,
    distance_to_agreement: int = 1,
    gamma_cap_value: float = 2,
    global_dose: bool = True,
    dose_threshold: float = 5,
    resolution_factor: int = 3,
    fill_value: float = np.nan,
) -> (np.ndarray, np.ndarray, np.ndarray):
    """Low et al. 1-D gamma of two profiles (reference core/gamma.py:333-460); a batch of one for ``gamma_1d_batch``.  Returns
    ``(gamma, eval_interp_array, eval_x_vals)``: the gamma of each reference point (``fill_value`` below ``dose_threshold`` % of the
    reference's maximum), and the evaluation interpolated at the ``int(DTA * resolution_factor * 2 + 1)`` search positions of each
    evaluated point, with those positions.

    The search positions and the interpolated evaluation are bit-identical to the reference.  The gamma values can differ from the
    reference's in the last bit: the reference squares the per-sample distance and dose with ``**2``, which Python and numpy hand to
    the C library's ``pow``, and glibc's ``pow(x, 2)`` is not always the correctly rounded ``x * x`` (about one square in a
    thousand differs by one unit in the last place); the device squares by multiplying.

    Divergence from the reference: float32 (or other non-float64 floating) coordinates raise ``TypeError`` (the reference computes
    their search positions in float32), and so does a reference whose dose criterion is neither float32 nor float64 (float16).
    """
    if _not_1d(reference, evaluation):
        raise _ndim_error(reference, evaluation)
    return gamma_1d_batch([reference], [evaluation], None if reference_coordinates is None else [reference_coordinates],
                          None if evaluation_coordinates is None else [evaluation_coordinates], dose_to_agreement,
                          distance_to_agreement, gamma_cap_value, global_dose, dose_threshold, resolution_factor, fill_value)[0]


def _pymin(a):
    """Python's min() over an array (its error when empty, its nan rules), by numpy where they agree"""
    return min(a) if a.size == 0 or (a.dtype.kind == "f" and np.isnan(a).any()) else a.min()


def _pymax(a):
    return max(a) if a.size == 0 or (a.dtype.kind == "f" and np.isnan(a).any()) else a.max()


def _prepare_1d(reference, evaluation, rc, ec, dose_to_agreement, distance_to_agreement, global_dose, dose_threshold,
                resolution_factor, num):
    """the reference's checks and O(n) preparation (core/gamma.py:392-429)"""
    if _not_1d(reference, evaluation):
        raise _ndim_error(reference, evaluation)
    if rc is None:
        rc = np.arange(len(reference), dtype=float)
    if len(reference) != len(rc):
        raise ValueError(f"Reference and reference_x_values must be the same length. Got reference: {len(reference)} and "
                         f"reference_x_values: {len(rc)}")
    if ec is None:
        ec = np.arange(len(evaluation), dtype=float)
    if len(evaluation) != len(ec):
        raise ValueError(f"Evaluation and evaluation_x_values must be the same length. Got evaluation: {len(evaluation)} and "
                         f"evaluation_x_values: {len(ec)}")
    if _pymin(ec) - 1 > _pymin(rc) or _pymax(ec) + 1 < _pymax(rc):
        raise ValueError("The reference x-values must be within the range of the evaluation x-values")
    if resolution_factor < 1 or not isinstance(resolution_factor, int):
        raise ValueError("Resolution factor must be an integer greater than 0")
    threshold = reference.max() / 100 * dose_threshold
    dose_ta = dose_to_agreement / 100 * reference.max()
    for c in (rc, ec):
        if c.dtype.kind == "f":
            _float64_coordinates(c)
    if np.result_type(dose_ta) not in (np.float32, np.float64):
        raise TypeError(f"the dose criterion of a {reference.dtype} reference is {np.result_type(dose_ta)}; float32 and float64 "
                        f"are supported")
    order = np.argsort(ec, kind="mergesort")                   # interp1d's sort of the evaluation
    mask = ~(reference < threshold)
    if mask.any() and num < 0:
        raise ValueError(f"Number of samples, {num}, must be non-negative.")
    if mask.any() and num == 0:
        raise ValueError("min() iterable argument is empty")
    if global_dose:
        dose_ta2 = np.full(int(mask.sum()), dose_ta ** 2, dtype=np.float64)
        single = np.result_type(dose_ta) == np.float32
    else:
        local = dose_to_agreement / 100 * reference[mask]
        # the reference's scalar ``dose_ta**2`` is libm pow / powf, which does not always round as local * local
        dose_ta2 = np.array([v ** 2 for v in local], dtype=np.float64)
        single = local.dtype == np.float32
    return (mask, ec[order].astype(np.float64), evaluation[order].astype(np.float64), rc[mask].astype(np.float64),
            reference[mask].astype(np.float64), dose_ta2, single)


def _gamma_list(n: int, mask: np.ndarray, g: np.ndarray, cap, fill_value) -> np.ndarray:
    """np.asarray of the reference's list: fill_value below the threshold, min(gamma, cap) -- the cap object or a Python float --
    elsewhere"""
    capped = g == cap
    probe = ([fill_value] if not mask.all() else []) + ([cap] if capped.any() else []) + ([1.0] if not capped.all() else [])
    if np.asarray(probe).dtype == np.float64:
        out = np.full(n, fill_value, dtype=np.float64)
        out[mask] = g
        return out
    items = [fill_value] * n
    for i, v, c in zip(np.flatnonzero(mask), g.tolist(), capped.tolist()):
        items[i] = cap if c else v
    return np.asarray(items)


def gamma_1d_batch(
    references,
    evaluations,
    reference_coordinates=None,
    evaluation_coordinates=None,
    dose_to_agreement: float = 1,
    distance_to_agreement: int = 1,
    gamma_cap_value: float = 2,
    global_dose: bool = True,
    dose_threshold: float = 5,
    resolution_factor: int = 3,
    fill_value: float = np.nan,
    *,
    ctx: nat.Context | None = None,
) -> list[tuple[np.ndarray, np.ndarray, np.ndarray]]:
    """``gamma_1d`` of n pairs of 1-D profiles, whose lengths may differ from pair to pair: ``references`` and ``evaluations`` are
    sequences of n arrays (a 2-D array is a sequence of rows), the coordinates None or one array (or None) per pair.  Returns the
    list of the n ``(gamma, eval_interp_array, eval_x_vals)``.  Every pair's arguments are checked, with the reference's exceptions,
    before one device call (one upload, one kernel, one download) computes them all."""
    refs, evs = _rows(references), _rows(evaluations)
    if len(refs) != len(evs):
        raise ValueError(f"{len(refs)} references but {len(evs)} evaluations")
    n = len(refs)
    rcs, ecs = _coordinate_rows(reference_coordinates, n), _coordinate_rows(evaluation_coordinates, n)
    num = int(distance_to_agreement * resolution_factor * 2 + 1)
    preps = [_prepare_1d(refs[i], evs[i], rcs[i], ecs[i], dose_to_agreement, distance_to_agreement, global_dose, dose_threshold,
                         resolution_factor, num) for i in range(n)]
    if n == 0:
        return []
    ctx = ctx or nat.Context.default()
    g, samples, xs = nat.gamma1d(
        ctx, _offsets([len(p[1]) for p in preps]), _offsets([len(p[3]) for p in preps]), [p[6] for p in preps],
        np.concatenate([p[1] for p in preps]), np.concatenate([p[2] for p in preps]), np.concatenate([p[3] for p in preps]),
        np.concatenate([p[4] for p in preps]), np.concatenate([p[5] for p in preps]), float(distance_to_agreement),
        float(distance_to_agreement ** 2), max(num, 1), float(gamma_cap_value))
    out, at = [], 0
    for ref, p in zip(refs, preps):
        k = len(p[3])
        out.append((_gamma_list(len(ref), p[0], g[at:at + k], gamma_cap_value, fill_value), samples[at:at + k].ravel(),
                    xs[at:at + k].ravel()))
        at += k
    return out
