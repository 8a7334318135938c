"""API-surface glue mirroring pylinac/core/utilities.py:27-110 (ResultBase, ResultsDataMixin, convert_to_enum)."""
from __future__ import annotations

import json
from abc import abstractmethod
from datetime import datetime
from enum import Enum
from typing import Generic, TypeVar

from pydantic import BaseModel, ConfigDict, Field

from ..version import __version__
from .warnings import WarningCollectorMixin


def convert_to_enum(value, enum: type[Enum]) -> Enum:
    """core/utilities.py:27-32"""
    if isinstance(value, enum):
        return value
    return enum(value)


class OptionListMixin:
    """core/utilities.py:35-45: ``options()`` lists the values of an enum-like class's public, non-callable attributes."""

    @classmethod
    def options(cls) -> list[str]:
        return [v for k, v in cls.__dict__.items() if not k.startswith("__") and not callable(v)]


class ResultBase(BaseModel):
    """core/utilities.py:48-66"""

    model_config = ConfigDict(arbitrary_types_allowed=True)
    pylinac_version: str = Field(default=__version__, title="Pylinac version")
    date_of_analysis: datetime = Field(default_factory=datetime.today, title="Date of Analysis")
    warnings: list[dict] = Field(title="Warnings", default_factory=list)


T = TypeVar("T")


class ResultsDataMixin(Generic[T], WarningCollectorMixin):
    """core/utilities.py:72-110"""

    @abstractmethod
    def _generate_results_data(self) -> T:
        pass

    def results_data(self, as_dict: bool = False, as_json: bool = False, by_alias: bool = False, exclude: set[str] | None = None):
        if as_dict and as_json:
            raise ValueError("Cannot return as both dict and JSON. Pick one.")
        data = self._generate_results_data()
        if hasattr(data, "warnings") and hasattr(self, "get_captured_warnings"):
            data.warnings = self.get_captured_warnings()
        if as_dict:
            return json.loads(data.model_dump_json(by_alias=by_alias, exclude=exclude))
        if as_json:
            return data.model_dump_json(by_alias=by_alias, exclude=exclude)
        return data
