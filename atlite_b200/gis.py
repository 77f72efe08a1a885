"""Shapes -> indicator matrix on the cutout grid, computed on the GPU.

Host-side mirror of the reference's ``compute_indicatormatrix`` (gis.py:104-145)
for the case the hot path needs: ``orig`` = the cells of a regular cutout grid
(cutout.py:355-376).  I[i, j] is the fraction of cell j covered by shape i, j in
``cutout.grid`` order (iy * nx + ix).  The areas come from libatlite_b200's
``atl_indicator_compute`` (csrc/indicator.cu); there is no CPU fallback.
``compute_intersectionmatrix`` mirrors the reference's function of that name
(gis.py:148-183) the same way through ``atl_intersection_compute``; it also
takes points and lines (``geometry_parts``).

Shapes may be given without shapely:
  * anything with ``__geo_interface__`` (shapely geometries, geopandas rows),
  * GeoJSON geometry dicts of type Polygon / MultiPolygon (or Feature /
    GeometryCollection of those),
  * an ``(N, 2)`` array-like: one exterior ring,
  * a list of such arrays: exterior followed by holes.
Collections: list/tuple, dict (values), pandas Series, geopandas GeoSeries /
GeoDataFrame (its geometry column).
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sp

from . import _lib


def _is_ring(obj):
    try:
        a = np.asarray(obj, dtype=np.float64)
    except (TypeError, ValueError):
        return False
    return a.ndim == 2 and a.shape[1] >= 2 and a.shape[0] >= 1


# part kinds of a geometry (ATL_PART_* in include/atlite_b200.h)
PART_EXTERIOR, PART_HOLE, PART_LINE, PART_POINTS = 0, 1, 2, 3


def _coords(c, what):
    """Coordinate list -> (N, 2) float64 (any z dropped); None when empty."""
    a = np.asarray(c, dtype=np.float64)
    if a.size == 0:
        return None
    if a.ndim == 1 and what == "point":
        a = a[None, :]
    if a.ndim != 2 or a.shape[1] < 2:
        raise ValueError(f"a {what} must be an (N, >=2) coordinate array")
    return np.ascontiguousarray(a[:, :2])


def _polygon_parts(coords):
    """GeoJSON Polygon coordinates -> [(PART_EXTERIOR | PART_HOLE, ring)], exterior first."""
    out = []
    for k, ring in enumerate(coords):
        a = _coords(ring, "polygon ring")
        if a is not None:
            out.append((PART_HOLE if k > 0 else PART_EXTERIOR, a))
    return out


def _line_parts(lines):
    return [(PART_LINE, a) for a in (_coords(c, "line") for c in lines) if a is not None]


def _point_parts(points):
    a = _coords(points, "point")
    return [] if a is None else [(PART_POINTS, a)]


_POLYGONAL = {"Polygon": _polygon_parts,
              "MultiPolygon": lambda c: [p for poly in c for p in _polygon_parts(poly)]}
_LINEAL_PUNTAL = {"LineString": lambda c: _line_parts([c]),
                  "LinearRing": lambda c: _line_parts([c]),  # shapely's closed line without interior
                  "MultiLineString": _line_parts,
                  "Point": _point_parts,
                  "MultiPoint": _point_parts}


def geometry_parts(geom, polygonal=False):
    """One shape -> list of (kind, (N, 2) float64 coordinates), kind one of PART_*.
    Reads GeoJSON / ``__geo_interface__`` Point, MultiPoint, LineString,
    MultiLineString, LinearRing, Polygon, MultiPolygon, Feature and
    GeometryCollection (the union of its parts); an (N, 2) array is one exterior
    ring, a list of them an exterior followed by holes.  ``None`` and empty
    geometries give no parts.  ``polygonal=True`` rejects the non-polygon types."""
    if geom is None:
        return []
    if hasattr(geom, "__geo_interface__"):
        geom = geom.__geo_interface__
    if isinstance(geom, dict):
        t = geom.get("type")
        if t == "Feature":
            return geometry_parts(geom.get("geometry"), polygonal)
        if t == "GeometryCollection":
            return [p for g in geom.get("geometries", []) for p in geometry_parts(g, polygonal)]
        if t in _POLYGONAL:
            return _POLYGONAL[t](geom["coordinates"])
        if t in _LINEAL_PUNTAL and not polygonal:
            return _LINEAL_PUNTAL[t](geom["coordinates"])
        need = "Polygon / MultiPolygon" if polygonal else "a GeoJSON geometry"
        raise ValueError(f"unsupported geometry type {t!r} (need {need})")
    if _is_ring(geom):
        return _polygon_parts([geom])
    if isinstance(geom, (list, tuple)) and all(_is_ring(r) for r in geom):
        return _polygon_parts(geom)
    raise TypeError(f"cannot interpret {type(geom).__name__} as a {'polygon' if polygonal else 'geometry'}")


def geometry_rings(geom):
    """One polygonal shape -> list of (ring (N,2) float64, is_hole)."""
    return [(a, kind == PART_HOLE) for kind, a in geometry_parts(geom, polygonal=True)]


def line_azimuth(geom):
    """``arctan2(start.x - end.x, start.y - end.y)`` of a line's first and last coordinate, in
    radians (the reference's ``get_azimuth``, convert.py:1333-1337).  Only a LineString or
    LinearRing has the single coordinate sequence that takes; any other geometry raises."""
    g = geom.__geo_interface__ if hasattr(geom, "__geo_interface__") else geom
    t = g.get("type") if isinstance(g, dict) else type(geom).__name__
    if t not in ("LineString", "LinearRing"):
        raise TypeError(f"a line azimuth needs a LineString or LinearRing, not {t}")
    xy = _coords(g["coordinates"], "line")
    if xy is None:
        raise ValueError("a line azimuth needs a non-empty line")
    return float(np.arctan2(xy[0, 0] - xy[-1, 0], xy[0, 1] - xy[-1, 1]))


def _iter_shapes(shapes):
    if hasattr(shapes, "columns") and hasattr(shapes, "geometry"):  # GeoDataFrame
        shapes = shapes.geometry
    if isinstance(shapes, dict):
        return list(shapes.values())
    if hasattr(shapes, "values") and not isinstance(shapes, np.ndarray):  # pandas / geopandas Series
        return list(shapes.values)
    return list(shapes)


def pack_shapes(shapes):
    """Collection of shapes -> (shape_ring_ptr, ring_ptr, ring_is_hole, xy) in the
    layout ``atl_indicator_compute`` takes (include/atlite_b200.h)."""
    shape_ring_ptr, ring_ptr, holes, chunks = [0], [0], [], []
    for g in _iter_shapes(shapes):
        for ring, hole in geometry_rings(g):
            chunks.append(ring)
            ring_ptr.append(ring_ptr[-1] + len(ring))
            holes.append(1 if hole else 0)
        shape_ring_ptr.append(len(holes))
    xy = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros((0, 2)), dtype=np.float64)
    return (np.asarray(shape_ring_ptr, dtype=np.int64), np.asarray(ring_ptr, dtype=np.int64),
            np.asarray(holes, dtype=np.int8), xy)


def pack_geometries(shapes):
    """Collection of shapes of any kind (see ``geometry_parts``) ->
    (shape_part_ptr, part_ptr, part_kind, xy) in the layout ``atl_intersection_compute``
    takes (include/atlite_b200.h)."""
    shape_part_ptr, part_ptr, kinds, chunks = [0], [0], [], []
    for g in _iter_shapes(shapes):
        for kind, a in geometry_parts(g):
            chunks.append(a)
            part_ptr.append(part_ptr[-1] + len(a))
            kinds.append(kind)
        shape_part_ptr.append(len(kinds))
    xy = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros((0, 2)), dtype=np.float64)
    return (np.asarray(shape_part_ptr, dtype=np.int64), np.asarray(part_ptr, dtype=np.int64),
            np.asarray(kinds, dtype=np.int8), xy)


def cell_edges(c):
    """(lo, hi) float64 edges of the cells about the centres ``c``, computed as the
    reference's ``Cutout.grid`` boxes are (cutout.py:369-372): c -/+ (c[1] - c[0]) / 2.
    On grids whose step is not dyadic neighbouring boxes overlap or leave a gap of an ulp."""
    c = np.asarray(c, dtype=np.float64)
    half = (c[1] - c[0]) / 2
    return np.ascontiguousarray(c - half), np.ascontiguousarray(c + half)


def regular_axis(c, name):
    """(first centre, step) of an ascending, evenly spaced coordinate."""
    c = np.asarray(c, dtype=np.float64)
    if c.ndim != 1 or len(c) < 1:
        raise ValueError(f"coordinate {name!r} must be 1-D and non-empty")
    if len(c) == 1:
        raise ValueError(f"coordinate {name!r} has a single value: the cell size is undefined")
    d = np.diff(c)
    step = (c[-1] - c[0]) / (len(c) - 1)
    if not step > 0 or not np.allclose(d, step, rtol=1e-6, atol=1e-9 * abs(step)):
        raise ValueError(f"coordinate {name!r} must be ascending and evenly spaced")
    return float(c[0]), float(step)


def compute_indicatormatrix(x, y, shapes, device=None):
    """CSR (n_shapes, len(y) * len(x)) of covered cell fractions for the regular
    grid with cell centres ``x`` (columns) and ``y`` (rows)."""
    from .engine import current_device

    lib = _lib.load()
    x0, dx = regular_axis(x, "x")
    y0, dy = regular_axis(y, "y")
    nx, ny = len(x), len(y)
    srp, rp, holes, xy = pack_shapes(shapes)
    n_shapes = len(srp) - 1
    h = C.c_void_p()
    device = current_device() if device is None else device
    _lib.check(lib.atl_indicator_compute(device, ny, nx, x0, dx, y0, dy, n_shapes, _lib.ptr(srp), _lib.ptr(rp),
                                         _lib.ptr(holes), _lib.ptr(xy), C.byref(h)))
    return _export_csr(lib, h, n_shapes, ny * nx)


def compute_intersectionmatrix(x, y, shapes, device=None):
    """CSR (n_shapes, len(y) * len(x)) with 1.0 where shape i intersects the closed
    box of cell j (gis.py:148-183 with ``orig`` = ``Cutout.grid``), j in
    ``cutout.grid`` order.  The boxes are the reference's float64 boxes
    (``cell_edges``) and the decision is exact (csrc/indicator.cu): a boundary
    contact counts.  Shapes may be points, lines, polygons or collections of them
    (``geometry_parts``); a shape that meets no cell gives an empty row."""
    from .engine import current_device

    lib = _lib.load()
    x0, dx = regular_axis(x, "x")
    y0, dy = regular_axis(y, "y")
    nx, ny = len(x), len(y)
    xlo, xhi = cell_edges(x)
    ylo, yhi = cell_edges(y)
    spp, pp, kinds, xy = pack_geometries(shapes)
    n_shapes = len(spp) - 1
    h = C.c_void_p()
    device = current_device() if device is None else device
    _lib.check(lib.atl_intersection_compute(device, ny, nx, x0, dx, y0, dy, _lib.ptr(xlo), _lib.ptr(xhi),
                                            _lib.ptr(ylo), _lib.ptr(yhi), n_shapes, _lib.ptr(spp), _lib.ptr(pp),
                                            _lib.ptr(kinds), _lib.ptr(xy), C.byref(h)))
    return _export_csr(lib, h, n_shapes, ny * nx)


def _export_csr(lib, h, n_shapes, n_cells):
    """AtlIndicator handle -> scipy CSR; frees the handle."""
    try:
        nnz = C.c_int64()
        _lib.check(lib.atl_indicator_nnz(h, C.byref(nnz)))
        indptr = np.empty(n_shapes + 1, dtype=np.int64)
        indices = np.empty(nnz.value, dtype=np.int32)
        data = np.empty(nnz.value, dtype=np.float64)
        _lib.check(lib.atl_indicator_export(h, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data)))
    finally:
        lib.atl_indicator_destroy(h)
    return sp.csr_matrix((data, indices, indptr), shape=(n_shapes, n_cells))


# land eligibility (gis.py:186-661 of the reference): availability.py
from .availability import (  # noqa: E402
    ExclusionContainer,
    Raster,
    compute_availabilitymatrix,
    padded_transform_and_shape,
    shape_availability,
)
