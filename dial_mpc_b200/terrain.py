"""Per-instance terrain: a heightfield under an instance's simulated robot and, when known, under its planner
(``dial_plan_set_instance_terrain``, include/dial_b200.h).

A terrain is a grid of fp32 heights ``h[j][i]`` (``nx`` x ``ny``, 2..``DIAL_MAXTERRAIN`` per side) with spacing
``s`` and origin ``(x0, y0)``: vertex (i, j) is the world point ``(x0 + i s, y0 + j s, h[j][i])``, heights in
absolute world z.  Each cell is split along its diagonal from (i, j) to (i+1, j+1) into two triangles, and
``height`` is the piecewise linear surface.  A floor contact's sphere (or capsule end) is tested against the
plane of the triangle under its centre; outside the grid the point is clamped into it and the plane is
horizontal.  The model is locally planar: it is accurate where the surface varies slowly at the scale of a
foot, as on slopes and rough ground, and does not represent steps or stairs (a sphere only sees the triangle
beneath its centre).

The generators build square grids centred on the world origin with a flat patch of radius ``flat_radius``
around it, so that an env's standing reset pose stays valid (reset states are not raised)."""
from __future__ import annotations

import ctypes as C
import dataclasses
import numbers
import os
from typing import Optional, Tuple

import numpy as np

from dial_mpc_b200 import _capi

MAXTERRAIN = _capi.DEFINES["DIAL_MAXTERRAIN"]
PLANT, PLANNER = _capi.DEFINES["DIAL_TERRAIN_PLANT"], _capi.DEFINES["DIAL_TERRAIN_PLANNER"]


@dataclasses.dataclass(frozen=True)
class Terrain:
    heights: np.ndarray               # [ny, nx] float32, world z
    spacing: float
    origin: Tuple[float, float]

    def c_struct(self) -> _capi.dial_terrain:
        """The ``dial_terrain`` of this grid; it points into ``heights``, which must outlive its use."""
        t = _capi.dial_terrain()
        t.ny, t.nx = self.heights.shape
        t.x0, t.y0 = self.origin
        t.spacing = self.spacing
        t.heights = self.heights.ctypes.data_as(C.c_void_p)
        return t


def plane(t: Terrain, x, y):
    """The plane of the triangle under the world points (x, y), in fp64: (H, sx, sy), the surface height there
    and the triangle's slopes; outside the grid the point is clamped into it and the slopes are 0."""
    h = np.asarray(t.heights, dtype=np.float64)
    ny, nx = h.shape
    s = float(t.spacing)
    u = (np.asarray(x, dtype=np.float64) - t.origin[0]) / s
    v = (np.asarray(y, dtype=np.float64) - t.origin[1]) / s
    inside = (u >= 0) & (u <= nx - 1) & (v >= 0) & (v <= ny - 1)
    u, v = np.clip(u, 0, nx - 1), np.clip(v, 0, ny - 1)
    i, j = np.minimum(u.astype(np.int64), nx - 2), np.minimum(v.astype(np.int64), ny - 2)
    fu, fv = u - i, v - j
    h00, h11 = h[j, i], h[j + 1, i + 1]
    lower = fu >= fv
    hm = np.where(lower, h[j, np.minimum(i + 1, nx - 1)], h[np.minimum(j + 1, ny - 1), i])
    a = np.where(lower, hm - h00, h11 - hm)
    b = np.where(lower, h11 - hm, hm - h00)
    return h00 + fu * a + fv * b, np.where(inside, a / s, 0.0), np.where(inside, b / s, 0.0)


def height(t: Terrain, x, y):
    """H(x, y): the terrain's surface height under the world points (x, y), in fp64."""
    return plane(t, x, y)[0]


def _square(size: float, spacing: float):
    if not (np.isfinite(size) and size > 0 and np.isfinite(spacing) and spacing > 0):
        raise ValueError(f"size and spacing must be finite and > 0, got {size!r}, {spacing!r}")
    n = int(round(size / spacing)) + 1
    if not 2 <= n <= MAXTERRAIN:
        raise ValueError(f"size / spacing gives {n} vertices per side, out of range (2..{MAXTERRAIN})")
    half = (n - 1) * spacing / 2
    xs = -half + spacing * np.arange(n)
    return n, (-half, -half), np.meshgrid(xs, xs)   # X[j, i], Y[j, i]


def rough(amplitude: float, wavelength: float, seed: int = 0, size: float = 10.0, spacing: float = 0.05,
          flat_radius: float = 0.5) -> Terrain:
    """Value noise: a seeded uniform lattice of heights in [-amplitude, amplitude] every ``wavelength`` metres,
    bilinearly interpolated at the grid's vertices.  Within ``flat_radius`` of the origin the ground is flat at
    z = 0, and the noise blends in over one wavelength beyond it.  Locally planar: no steps."""
    if not (np.isfinite(amplitude) and amplitude >= 0 and np.isfinite(wavelength) and wavelength > 0):
        raise ValueError(f"amplitude must be finite and >= 0 and wavelength finite and > 0, got {amplitude!r}, {wavelength!r}")
    n, origin, (X, Y) = _square(size, spacing)
    m = int(np.ceil(size / wavelength)) + 2
    lat = np.random.default_rng(seed).uniform(-amplitude, amplitude, (m, m))
    u, v = (X - origin[0]) / wavelength, (Y - origin[1]) / wavelength
    i, j = np.minimum(u.astype(np.int64), m - 2), np.minimum(v.astype(np.int64), m - 2)
    fu, fv = u - i, v - j
    h = ((1 - fu) * (1 - fv) * lat[j, i] + fu * (1 - fv) * lat[j, i + 1] + (1 - fu) * fv * lat[j + 1, i]
         + fu * fv * lat[j + 1, i + 1])
    blend = np.clip((np.hypot(X, Y) - flat_radius) / wavelength, 0.0, 1.0)
    return Terrain(np.ascontiguousarray(h * blend, dtype=np.float32), float(spacing), origin)


def slope(angle_deg: float, heading_deg: float = 0.0, size: float = 10.0, spacing: float = 0.05,
          flat_radius: float = 0.5) -> Terrain:
    """A ramp rising at ``angle_deg`` towards the heading ``heading_deg`` (0: +x) beyond the edge of the flat
    patch, and falling at the same angle behind it: z = tan(angle) (d - clip(d, -r, r)) with d the distance
    along the heading and r = ``flat_radius``.  With r = 0 it is one plane through the origin.  Locally planar:
    no steps."""
    if not (np.isfinite(angle_deg) and -80 <= angle_deg <= 80 and np.isfinite(heading_deg)):
        raise ValueError(f"angle_deg must be in -80..80 and heading_deg finite, got {angle_deg!r}, {heading_deg!r}")
    n, origin, (X, Y) = _square(size, spacing)
    psi = np.deg2rad(heading_deg)
    d = X * np.cos(psi) + Y * np.sin(psi)
    h = np.tan(np.deg2rad(angle_deg)) * (d - np.clip(d, -flat_radius, flat_radius))
    return Terrain(np.ascontiguousarray(h, dtype=np.float32), float(spacing), origin)


def grid(heights, spacing: float, origin=(0.0, 0.0)) -> Terrain:
    """A user grid: ``heights`` [ny, nx] (an array, nested lists or the path of a ``.npy`` file), vertex (i, j) at
    (origin[0] + i spacing, origin[1] + j spacing, heights[j][i])."""
    if isinstance(heights, (str, os.PathLike)):
        heights = np.load(heights)
    h = np.ascontiguousarray(heights, dtype=np.float32)
    if h.ndim != 2 or not (2 <= h.shape[0] <= MAXTERRAIN and 2 <= h.shape[1] <= MAXTERRAIN):
        raise ValueError(f"heights must be a [ny, nx] grid with 2..{MAXTERRAIN} per side, got shape {h.shape}")
    if not np.isfinite(h).all():
        raise ValueError("heights must be finite")
    if not (_real(spacing) and np.isfinite(spacing) and spacing > 0):
        raise ValueError(f"spacing must be a finite number > 0, got {spacing!r}")
    if not (len(origin) == 2 and all(_real(o) and np.isfinite(o) for o in origin)):
        raise ValueError(f"origin must be two finite numbers, got {origin!r}")
    return Terrain(h, float(spacing), (float(origin[0]), float(origin[1])))


def _real(x):
    return isinstance(x, numbers.Real) and not isinstance(x, bool)


@dataclasses.dataclass(frozen=True)
class TerrainSetting:
    """An instance's terrain: under its plant, and under its planner too when ``planner``."""
    terrain: Terrain
    planner: bool


_KINDS = {"rough": (rough, ("amplitude", "wavelength"), ("seed", "size", "spacing", "flat_radius")),
          "slope": (slope, ("angle",), ("heading", "size", "spacing", "flat_radius")),
          "grid": (grid, ("heights", "spacing"), ("origin",))}
_RENAME = {"angle": "angle_deg", "heading": "heading_deg"}


def terrain_setting(spec, sys=None) -> TerrainSetting:
    """A terrain spec -> the ``TerrainSetting`` of one instance.  The spec maps ``kind`` (``rough``, ``slope`` or
    ``grid``) and that kind's fields: rough ``amplitude``, ``wavelength`` [m], ``seed``; slope ``angle``,
    ``heading`` [deg]; both ``size``, ``spacing`` [m] and ``flat_radius``; grid ``heights`` (a [ny, nx] list or
    a ``.npy`` path), ``spacing`` and ``origin``.  ``planner: true`` lets the planner plan on the same terrain
    (perceptive); the default ``false`` keeps it on the flat floor (blind).  ``sys`` (optional): the model, which
    must have a floor pair.  Raises ValueError naming the bad entry."""
    if not isinstance(spec, dict) or spec.get("kind") not in _KINDS:
        raise ValueError(f"a terrain spec is a mapping with kind {' | '.join(_KINDS)}, got {spec!r}")
    fn, need, opt = _KINDS[spec["kind"]]
    extra = set(spec) - {"kind", "planner"} - set(need) - set(opt)
    if extra:
        raise ValueError(f"a {spec['kind']} terrain takes {', '.join(need + opt)} and planner, got {sorted(extra)[0]!r}")
    missing = [k for k in need if k not in spec]
    if missing:
        raise ValueError(f"a {spec['kind']} terrain needs {missing[0]!r}")
    planner = spec.get("planner", False)
    if not isinstance(planner, bool):
        raise ValueError(f"planner must be true or false, got {planner!r}")
    kw = {_RENAME.get(k, k): v for k, v in spec.items() if k not in ("kind", "planner")}
    for k, v in kw.items():
        if k == "seed" and not (isinstance(v, numbers.Integral) and not isinstance(v, bool)):
            raise ValueError(f"seed must be an int, got {v!r}")
        if k not in ("heights", "origin", "seed") and not _real(v):
            raise ValueError(f"{k} must be a number, got {v!r}")
    if sys is not None and not has_floor(sys):
        raise ValueError("the model has no floor pair (a plane geom on the world body against a sphere or capsule)")
    return TerrainSetting(fn(**kw), planner)


def has_floor(sys) -> bool:
    """Whether the model has a floor pair: a plane geom on the world body against a sphere or capsule."""
    md = _capi.fill_model_desc(getattr(sys, "model", sys))
    return any(md.pair_kind[k] in (0, 1) and md.geom_bodyid[md.pair_geom1[k]] == 0 for k in range(md.npair))


def terrains(setting: Optional[TerrainSetting]):
    """The (plant, planner) terrains of a setting; None: the flat floor."""
    if setting is None:
        return None, None
    return setting.terrain, setting.terrain if setting.planner else None
