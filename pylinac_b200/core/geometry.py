"""Host-side scalar geometry helpers (mirror of the parts of pylinac/core/geometry.py the hot path uses:
Point :70-224, Line :497-584).  Scalar work stays in Python (SURVEY.md section 2 row 12)."""
from __future__ import annotations

import math
from collections.abc import Iterable

import numpy as np


class Point:
    """core/geometry.py:70-224 (the subset used on the hot path)."""

    def __init__(self, x=0, y=0, z=0, idx=None, value=None, as_int: bool = False):
        if isinstance(x, Point):
            x, y, z, idx, value = x.x, x.y, x.z, x.idx, x.value
        elif isinstance(x, Iterable) and not isinstance(x, (str, bytes)):
            seq = list(x)
            x = seq[0] if len(seq) > 0 else 0
            y = seq[1] if len(seq) > 1 else y
            z = seq[2] if len(seq) > 2 else z
        if as_int:
            x, y, z = int(round(x)), int(round(y)), int(round(z))
        self.x, self.y, self.z, self.idx, self.value = x, y, z, idx, value

    def distance_to(self, thing) -> float:
        p = Point(thing)
        return math.sqrt((self.x - p.x) ** 2 + (self.y - p.y) ** 2 + (self.z - p.z) ** 2)

    def as_array(self, coords=("x", "y", "z")) -> np.ndarray:
        return np.array([getattr(self, c) for c in coords])

    def __add__(self, other):
        o = Point(other)
        return Point(self.x + o.x, self.y + o.y, self.z + o.z)

    def __sub__(self, other):
        o = Point(other)
        return Point(self.x - o.x, self.y - o.y, self.z - o.z)

    def __eq__(self, other):
        o = Point(other)
        return self.x == o.x and self.y == o.y and self.z == o.z

    _attr_list = ("x", "y", "z", "idx", "value")

    def __mul__(self, other):
        """IN PLACE, like the reference (core/geometry.py:190-196): every attribute that can be multiplied is, self is returned."""
        for attr in self._attr_list:
            try:
                setattr(self, attr, getattr(self, attr) * other)
            except TypeError:
                pass
        return self

    def __truediv__(self, other):
        """IN PLACE (core/geometry.py:198-204)"""
        for attr in self._attr_list:
            val = getattr(self, attr)
            if val is not None:
                setattr(self, attr, val / other)
        return self

    def __repr__(self):
        return f"Point(x={self.x:3.2f}, y={self.y:3.2f}, z={self.z:3.2f})"


class Vector:
    """core/geometry.py:408-480 (x, y, z triple with scalar length and component arithmetic)."""

    def __init__(self, x: float = 0, y: float = 0, z: float = 0):
        self.x, self.y, self.z = x, y, z

    def as_scalar(self) -> float:
        return math.sqrt(self.x**2 + self.y**2 + self.z**2)

    def as_point(self) -> Point:
        return Point(self.x, self.y, self.z)

    def dict(self) -> dict:
        return {"x": self.x, "y": self.y, "z": self.z}

    def distance_to(self, thing) -> float:
        p = Point(thing)
        return math.sqrt((self.x - p.x) ** 2 + (self.y - p.y) ** 2 + (self.z - p.z) ** 2)

    def __sub__(self, other):
        return Vector(self.x - other.x, self.y - other.y, self.z - other.z)

    def __add__(self, other):
        return Vector(self.x + other.x, self.y + other.y, self.z + other.z)

    def __neg__(self):
        return Vector(-self.x, -self.y, -self.z)

    def __truediv__(self, k: float):
        return Vector(self.x / k, self.y / k, self.z / k)

    def __mul__(self, k: float):
        return Vector(self.x * k, self.y * k, self.z * k)

    def __repr__(self):
        return f"Vector(x={self.x:.2f}, y={self.y:.2f}, z={self.z:.2f})"


class Line:
    """core/geometry.py:497-584"""

    def __init__(self, point1, point2):
        self.point1 = Point(point1)
        self.point2 = Point(point2)

    @property
    def m(self) -> float:
        return (self.point1.y - self.point2.y) / (self.point1.x - self.point2.x)

    @property
    def b(self) -> float:
        return self.point1.y - (self.m * self.point1.x)

    def y(self, x) -> float:
        return self.m * x + self.b

    def x(self, y) -> float:
        return (y - self.b) / self.m

    @property
    def center(self) -> Point:
        mid_x = np.abs((self.point2.x - self.point1.x) / 2 + self.point1.x)
        mid_y = (self.point2.y - self.point1.y) / 2 + self.point1.y
        return Point(mid_x, mid_y)

    @property
    def length(self) -> float:
        return self.point1.distance_to(self.point2)

    def distance_to(self, point) -> float:
        point = Point(point).as_array()
        lp1 = self.point1.as_array()
        lp2 = self.point2.as_array()
        numerator = np.sqrt(np.sum(np.power(np.cross((lp2 - lp1), (lp1 - point)), 2)))
        denominator = np.sqrt(np.sum(np.power(lp2 - lp1, 2)))
        return numerator / denominator


class Circle:
    """core/geometry.py:213-405 (centre, radius, area, diameter, as_dict; plotting is out of scope)."""

    def __init__(self, center_point=None, radius: float | None = None):
        if center_point is None:
            center_point = Point()
        elif isinstance(center_point, Point) or (isinstance(center_point, Iterable) and not isinstance(center_point, (str, bytes))):
            center_point = Point(center_point)
        else:
            raise TypeError("Circle center must be of type Point or iterable")
        self.center = center_point
        self.radius = radius

    @property
    def area(self) -> float:
        return math.pi * self.radius**2

    @property
    def diameter(self) -> float:
        return self.radius * 2

    def as_dict(self) -> dict:
        return {"center_x": self.center.x, "center_y": self.center.y, "diameter": self.diameter}


class Rectangle:
    """core/geometry.py:632-723.  Image coordinates (+x right, +y down); ``rotation`` in degrees, positive = clockwise on screen.
    ``vertices`` = [TL, TR, BR, BL] of the UNROTATED rectangle, rotated about the origin and then translated to ``center`` (the
    reference composes skimage's ``EuclideanTransform(rotation, translation)``: x' = x cos - y sin + tx, y' = x sin + y cos + ty)."""

    def __init__(self, width: float, height: float, center, rotation: float = 0.0):
        if not width > 0 or not height > 0:
            raise ValueError("Rectangle width and height must be positive")
        self.width = width
        self.height = height
        self.center = Point(center)
        self.rotation = rotation

    @property
    def area(self) -> float:
        return self.width * self.height

    @property
    def vertices(self) -> list[Point]:
        half = np.array([[-1, -1], [1, -1], [1, 1], [-1, 1]]) @ np.diag((self.width, self.height)) / 2
        a = np.deg2rad(self.rotation)
        rot = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]])
        pts = half @ rot.T + self.center.as_array(("x", "y"))
        return [Point(p) for p in pts]

    @property
    def tl_corner(self) -> Point:
        return self.vertices[0]

    @property
    def tr_corner(self) -> Point:
        return self.vertices[1]

    @property
    def br_corner(self) -> Point:
        return self.vertices[2]

    @property
    def bl_corner(self) -> Point:
        return self.vertices[3]


def direction_to_coords(start_x: float, start_y: float, distance: float, angle_degrees: float) -> tuple[float, float]:
    """core/geometry.py:43-67: the point `distance` from (start_x, start_y) at `angle_degrees` (0 pointing right, i.e. the unit
    circle)"""
    angle_radians = math.radians(angle_degrees)
    return start_x + distance * math.cos(angle_radians), start_y + distance * math.sin(angle_radians)
