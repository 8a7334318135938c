"""Warning capture for the analysis classes -- the contract of ``pylinac/core/warnings.py:13-112``.

Every public method of a class decorated with :func:`capture_warnings` runs inside ``warnings.catch_warnings(record=True)``; what
it emits is stored on the instance (message, category, filename, lineno, line), re-emitted so it stays visible, and reported by
``results_data().warnings`` (deduplicated).  Nested decorated calls are captured once, by the outermost call.
"""
from __future__ import annotations

import functools
import sys
import threading
import types
import warnings as _warnings

_FIELDS = ("message", "category", "filename", "lineno", "line")


def _describe(w) -> dict:
    return {"message": str(w.message), "category": w.category.__name__, "filename": w.filename, "lineno": w.lineno, "line": w.line}


class WarningCollectorMixin:
    """Per-instance store of captured warnings (core/warnings.py:13-42)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._ensure_store()

    def _ensure_store(self) -> None:
        # the analysis classes here do not all chain to super().__init__(): create the store lazily
        if "_captured_warnings" not in self.__dict__:
            self._captured_warnings = []
            self._warnings_lock = threading.Lock()
            self._in_warning_capture = False

    def _add_warnings(self, items: list[dict]) -> None:
        self._ensure_store()
        with self._warnings_lock:
            self._captured_warnings.extend(items)

    def get_captured_warnings(self) -> list[dict]:
        self._ensure_store()
        with self._warnings_lock:
            seen, out = set(), []
            for w in self._captured_warnings:
                key = tuple(sorted(w.items(), key=lambda kv: kv[0]))
                if key not in seen:
                    seen.add(key)
                    out.append(w)
            return out

    def clear_captured_warnings(self) -> None:
        self._ensure_store()
        with self._warnings_lock:
            self._captured_warnings.clear()


def capture_warnings_method_wrapper(method):
    """core/warnings.py:45-88"""

    @functools.wraps(method)
    def wrapper(self, *args, **kwargs):
        if getattr(self, "_in_warning_capture", False):
            return method(self, *args, **kwargs)
        self._in_warning_capture = True
        try:
            with _warnings.catch_warnings(record=True) as caught:
                _warnings.simplefilter("always")
                result = method(self, *args, **kwargs)
                items = [_describe(w) for w in caught]
            if hasattr(self, "_add_warnings"):
                self._add_warnings(items)
            for w in caught:   # keep them visible on the console
                _warnings.showwarning(message=w.message, category=w.category, filename=w.filename, lineno=w.lineno, file=sys.stderr,
                                      line=w.line)
            return result
        finally:
            self._in_warning_capture = False

    return wrapper


def capture_warnings(cls):
    """Class decorator (core/warnings.py:91-112): wrap the methods defined on ``cls`` and the public methods it inherits."""
    is_func = lambda a: isinstance(a, (types.FunctionType, types.MethodType))  # noqa: E731
    own = dict(cls.__dict__)
    for name, attr in own.items():
        if is_func(attr):
            setattr(cls, name, capture_warnings_method_wrapper(attr))
    for parent in cls.__mro__[1:]:
        if parent is object:
            continue
        for name, attr in parent.__dict__.items():
            # the live dict: the first class of the MRO that defines a method wins, as in attribute lookup
            if name.startswith("_") or name in cls.__dict__:
                continue
            if is_func(attr):
                setattr(cls, name, capture_warnings_method_wrapper(attr))
    return cls
