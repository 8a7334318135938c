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
