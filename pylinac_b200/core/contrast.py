"""Contrast definitions (core/contrast.py): ``Contrast`` and ``visibility``, ``contrast``, ``rms``, ``difference``, ``michelson``,
``weber``, ``ratio``, with the reference's signatures, results, warnings and exceptions.

These are host arithmetic on a handful of values (a disk's median and a background value), evaluated with the numpy / Python
operations the reference uses, so that the results, numpy's warnings and the exceptions are the same: a zero float64 background
gives numpy's ``inf`` / ``nan`` and its RuntimeWarning, a zero Python-float background Python's ZeroDivisionError."""
from __future__ import annotations

import numpy as np

from .utilities import OptionListMixin


class Contrast(OptionListMixin):
    """Contrast calculation technique. See :ref:`visibility`."""

    MICHELSON = "Michelson"  #:
    WEBER = "Weber"  #:
    RATIO = "Ratio"  #:
    RMS = "Root Mean Square"  #:
    DIFFERENCE = "Difference"  #:


# The reference's message for an unknown method lists its Contrast class dictionary; the text is kept so that code matching on it works.
_OPTIONS_TEXT = "dict_values({!r})".format(["pylinac.core.contrast", Contrast.__doc__, Contrast.MICHELSON, Contrast.WEBER, Contrast.RATIO,
                                             Contrast.RMS, Contrast.DIFFERENCE])


RMS_RANGE_MESSAGE = "RMS calculations require the input array to be normalized. I.e. only values between 0 and 1."


def visibility(array: np.ndarray, radius: float, std: float, algorithm: str) -> float:
    """The Rose model of the visual perception of CNR: ``contrast(array, algorithm) * sqrt(pi * radius**2) / std``.  Not meant for
    high-contrast objects."""
    return contrast(array, algorithm) * np.sqrt(radius**2 * np.pi) / std


def _pair(array: np.ndarray, algorithm: str) -> tuple:
    if array.size != 2:
        raise ValueError(f"For {algorithm} algorithm, the array must be exactly 2 elements. Consult the ``{algorithm.lower()}`` "
                         "function for parameter details")
    return array[0], array[1]


def contrast(array: np.ndarray, algorithm: str) -> float:
    """The contrast of `array` by `algorithm` (a ``Contrast`` value, any case).  Michelson and RMS take any array; Weber, Ratio and
    Difference take (feature, background)."""
    method = algorithm.lower()
    if method == Contrast.MICHELSON.lower():
        return michelson(array)
    if method == Contrast.WEBER.lower():
        return weber(*_pair(array, "Weber"))
    if method == Contrast.RMS.lower():
        return rms(array)
    if method == Contrast.RATIO.lower():
        return ratio(*_pair(array, "Ratio"))
    if method == Contrast.DIFFERENCE.lower():
        return difference(*_pair(array, "Difference"))
    raise ValueError(f"Contrast input of {method} did not match any valid options: {_OPTIONS_TEXT}")


def rms(array: np.ndarray) -> float:
    """The root-mean-square contrast, the population std of `array`; its values must lie within [0, 1]."""
    if array.min() < 0 or array.max() > 1:
        raise ValueError(RMS_RANGE_MESSAGE)
    return np.sqrt(np.mean((array - array.mean()) ** 2))


def difference(feature: float, background: float) -> float:
    """|feature - background|"""
    return abs(feature - background)


def michelson(array: np.ndarray) -> float:
    """(max - min) / (max + min) of `array`, NaN ignored."""
    hi, lo = np.nanmax(array), np.nanmin(array)
    return (hi - lo) / (hi + lo)


def weber(feature: float, background: float) -> float:
    """|feature - background| / background (the absolute difference, as the reference keeps for backwards compatibility)."""
    return abs(feature - background) / background


def ratio(feature: float, reference: float) -> float:
    """feature / reference"""
    return feature / reference
