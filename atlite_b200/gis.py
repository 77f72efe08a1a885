"""Shapes -> indicator matrix, computed on the GPU.

Host-side mirror of the reference's ``compute_indicatormatrix`` (gis.py:104-145) in two
forms.  The grid form takes ``orig`` as the cells of a regular cutout grid
(cutout.py:355-376): I[i, j] is the fraction of cell j covered by shape i, j in
``cutout.grid`` order (iy * nx + ix), from libatlite_b200's ``atl_indicator_compute``
(csrc/indicator.cu).  The overlay form takes two polygon collections, as the reference
does, through ``atl_overlay_compute`` (csrc/overlay.cu).  There is no CPU fallback.
``compute_intersectionmatrix`` mirrors the reference's function of that name
(gis.py:148-183) in the same two forms: the grid form through
``atl_intersection_compute`` (csrc/indicator.cu), and the general form, any two
geometry collections, through ``atl_intersects_compute`` (csrc/overlay.cu).  Both
take points, lines and polygons (``geometry_parts``).

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
import math

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


def pack_geometries(shapes, polygonal=False):
    """Collection of shapes of any kind (see ``geometry_parts``) ->
    (shape_part_ptr, part_ptr, part_kind, xy) in the layout ``atl_intersection_compute``
    takes (include/atlite_b200.h).  ``polygonal=True`` rejects the non-polygon types: then
    every kind is PART_EXTERIOR (0) or PART_HOLE (1), and the arrays are the
    (shape_ring_ptr, ring_ptr, ring_is_hole, xy) that ``atl_indicator_compute`` and
    ``atl_overlay_compute`` take."""
    shape_part_ptr, part_ptr, kinds, chunks = [0], [0], [], []
    for g in _iter_shapes(shapes):
        for kind, a in geometry_parts(g, polygonal):
            chunks.append(a)
            part_ptr.append(part_ptr[-1] + len(a))
            kinds.append(kind)
        shape_part_ptr.append(len(kinds))
    xy = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros((0, 2)), dtype=np.float64)
    return (np.asarray(shape_part_ptr, dtype=np.int64), np.asarray(part_ptr, dtype=np.int64),
            np.asarray(kinds, dtype=np.int8), xy)


def pack_shapes(shapes):
    """Polygonal shapes -> (shape_ring_ptr, ring_ptr, ring_is_hole, xy): ``pack_geometries(shapes, polygonal=True)``."""
    return pack_geometries(shapes, polygonal=True)


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


def _numeric_1d(obj):
    """``obj`` as a 1-D NumPy array of numbers (a coordinate such as ``cutout.coords["x"]``), else None."""
    if obj is None or isinstance(obj, dict) or hasattr(obj, "__geo_interface__") or hasattr(obj, "geometry"):
        return None
    try:
        a = np.asarray(obj)
    except (TypeError, ValueError):
        return None
    return a if a.ndim == 1 and a.dtype.kind in "iuf" else None


def _is_crs(v):
    return v is None or isinstance(v, (int, np.integer, str)) or hasattr(v, "to_epsg") or hasattr(v, "to_authority")


def _grid_form(args, kwargs):
    """Whether a ``compute_indicatormatrix`` or ``compute_intersectionmatrix`` call takes the grid form (see
    ``compute_indicatormatrix``'s docstring)."""
    if "x" in kwargs or "shapes" in kwargs:
        return True
    a = _numeric_1d(args[0] if args else kwargs.get("orig"))
    if a is None:
        return False
    if a.size:
        return True
    # an empty sequence: an empty orig collection, unless a third positional argument that is no
    # CRS shows that it is an empty grid axis (which the grid form then refuses)
    return len(args) > 2 and not _is_crs(args[2])


def compute_indicatormatrix(*args, **kwargs):
    """Area overlap matrix of shapes, in one of two forms, chosen by the arguments.

    Grid form, when the first argument is a non-empty 1-D array-like of numbers (as
    ``cutout.coords["x"]`` is), or is passed as ``x=``, or ``shapes=`` is given:
    ``compute_indicatormatrix(x, y, shapes, device=None)`` returns the CSR (n_shapes, len(y) *
    len(x)) of covered cell fractions for the regular grid with cell centres ``x`` (columns) and
    ``y`` (rows).  An empty first argument is read as an empty grid axis (and refused as such) only
    when the third positional argument is not a CRS.

    Overlay form, otherwise: ``compute_indicatormatrix(orig, dest, orig_crs=4326, dest_crs=4326,
    device=None)`` returns the CSR (len(dest), len(orig)) with I[i, j] = area(dest_i ∩ orig_j) /
    area(orig_j), as the reference's function (gis.py:104-145); see ``overlay_indicatormatrix``.
    An empty ``orig`` gives a matrix with no columns."""
    if _grid_form(args, kwargs):
        return _grid_indicatormatrix(*args, **kwargs)
    return overlay_indicatormatrix(*args, **kwargs)


def _ring_shape_areas(srp, rp, holes, xy):
    """Planar area of every packed shape: exteriors minus holes (orientation free)."""
    n_shapes, n_rings = len(srp) - 1, len(rp) - 1
    if n_rings == 0:
        return np.zeros(n_shapes)
    ring_of = np.repeat(np.arange(n_rings), np.diff(rp))
    first = xy[rp[:-1]][ring_of]
    nxt = np.arange(len(xy)) + 1
    nxt[rp[1:] - 1] = rp[:-1]  # the last vertex of a ring closes onto its first
    a, b = xy - first, xy[nxt] - first
    area2 = np.bincount(ring_of, weights=a[:, 0] * b[:, 1] - b[:, 0] * a[:, 1], minlength=n_rings)
    ring_area = np.abs(area2) / 2 * np.where(holes != 0, -1.0, 1.0)
    return np.bincount(np.repeat(np.arange(n_shapes), np.diff(srp)), weights=ring_area, minlength=n_shapes)


def _crs_pair(orig_crs, dest_crs):
    """None when the two CRSs are equal by ``_crs_key`` (the vertices stay as they are), else the
    (dest, orig) ``proj.epsg`` keys; ``NotImplementedError`` when either is outside
    ``proj.SUPPORTED``."""
    from . import proj

    if _crs_key(orig_crs) == _crs_key(dest_crs):
        return None
    return proj.epsg(dest_crs), proj.epsg(orig_crs)


def _dest_into_orig(d_xy, pair):
    """Packed dest vertices projected into the orig CRS (``_crs_pair``), edges straight; ``ValueError``
    for a vertex without an image."""
    from .availability import _project

    if pair is None or not len(d_xy):
        return d_xy
    return np.ascontiguousarray(_project(d_xy, *pair))


def overlay_indicatormatrix(orig, dest, orig_crs=4326, dest_crs=4326, device=None):
    """CSR (len(dest), len(orig)) float64 with I[i, j] = area(dest_i ∩ orig_j) / area(orig_j), the
    reference's ``compute_indicatormatrix(orig, dest, orig_crs, dest_crs)`` (gis.py:104-145) for two
    polygon collections, computed on the GPU (csrc/overlay.cu).  Columns are ascending within each
    row and the result is bitwise repeatable.

    ``orig`` and ``dest``: collections of Polygon / MultiPolygon shapes in any form this module
    reads (shapely or ``__geo_interface__`` objects, GeoJSON dicts, (N, 2) rings, lists of rings,
    Series, GeoSeries, GeoDataFrame); other geometry types raise ``ValueError``.  An empty or
    ``None`` shape gives an empty row (dest) or column (orig); an orig shape with rings but zero
    area raises ``ValueError``.  Areas are planar, in ``orig_crs`` units; fractions <= 1e-10 are not
    stored and shapes that only touch give no entry.  Parts of one shape that overlap count twice.

    CRSs are compared by their key (``proj.epsg`` where it applies): equal CRSs leave every vertex
    as it is, whatever they are.  Otherwise both must be in ``proj.SUPPORTED``
    (``NotImplementedError``), and the dest vertices are projected into ``orig_crs`` with straight
    edges (``ValueError`` for a vertex without an image).  The geometries' own ``.crs`` is not
    read.  Every argument is checked before any device work.  Semantics and deviations: DESIGN.md
    section 1."""
    from .engine import current_device

    pair = _crs_pair(orig_crs, dest_crs)
    o_srp, o_rp, o_holes, o_xy = pack_shapes(orig)
    d_srp, d_rp, d_holes, d_xy = pack_shapes(dest)
    d_xy = _dest_into_orig(d_xy, pair)
    area = _ring_shape_areas(o_srp, o_rp, o_holes, o_xy)
    bad = np.flatnonzero((np.diff(o_srp) > 0) & ~(area > 0))
    if len(bad):
        raise ValueError(f"orig shape at position {int(bad[0])} has zero area")
    n_orig, n_dest = len(o_srp) - 1, len(d_srp) - 1
    lib = _lib.load()
    h = C.c_void_p()
    device = current_device() if device is None else device
    _lib.check(lib.atl_overlay_compute(device, n_orig, _lib.ptr(o_srp), _lib.ptr(o_rp), _lib.ptr(o_holes),
                                       _lib.ptr(o_xy), n_dest, _lib.ptr(d_srp), _lib.ptr(d_rp), _lib.ptr(d_holes),
                                       _lib.ptr(d_xy), C.byref(h)))
    return _export_csr(lib, h, n_dest, n_orig)


def _grid_indicatormatrix(x, y, shapes, device=None):
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


def compute_intersectionmatrix(*args, **kwargs):
    """Intersection matrix of shapes, in one of two forms, chosen by the arguments as
    ``compute_indicatormatrix`` chooses (``_grid_form``).

    Grid form: ``compute_intersectionmatrix(x, y, shapes, device=None)`` returns the CSR (n_shapes,
    len(y) * len(x)) with 1.0 where shape i meets the closed box of cell j; see
    ``_grid_intersectionmatrix``.

    General form, otherwise: ``compute_intersectionmatrix(orig, dest, orig_crs=4326, dest_crs=4326,
    device=None)`` returns the CSR (len(dest), len(orig)) with 1.0 where dest_i and orig_j intersect,
    as the reference's function (gis.py:148-183); see ``shapes_intersectionmatrix``."""
    if _grid_form(args, kwargs):
        return _grid_intersectionmatrix(*args, **kwargs)
    return shapes_intersectionmatrix(*args, **kwargs)


def _grid_intersectionmatrix(x, y, shapes, device=None):
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


def shapes_intersectionmatrix(orig, dest, orig_crs=4326, dest_crs=4326, device=None):
    """CSR (len(dest), len(orig)) float64 with 1.0 where dest_i and orig_j intersect as closed sets
    (shapely ``intersects``: a boundary contact counts), the reference's
    ``compute_intersectionmatrix(orig, dest, orig_crs, dest_crs)`` (gis.py:148-183) for two geometry
    collections, computed on the GPU (csrc/overlay.cu).  Columns are ascending within each row and
    the result, sparsity pattern included, is bitwise repeatable.

    ``orig`` and ``dest``: collections of shapes of any kind ``pack_geometries`` reads (points,
    lines, polygons, their multi forms and collections; shapely or ``__geo_interface__`` objects,
    GeoJSON dicts, (N, 2) rings, Series, GeoSeries, GeoDataFrame).  An empty or ``None`` shape gives
    an empty row (dest) or column (orig), and each orig shape gets its own column.  The point set of
    a shape is every segment of its parts (ring edges with the closing edge, line segments, points)
    and the even-odd interior of each polygon (an exterior with the holes that follow it); a shape
    is the union of its polygons.  The decision is exact.

    CRSs are handled as in ``overlay_indicatormatrix``: equal CRSs leave every vertex as it is;
    otherwise both must be in ``proj.SUPPORTED`` (``NotImplementedError``) and the dest vertices are
    projected into ``orig_crs`` with straight edges (``ValueError`` for a vertex without an image).
    Every argument is checked before any device work.  Semantics and deviations: DESIGN.md
    section 1."""
    from .engine import current_device

    pair = _crs_pair(orig_crs, dest_crs)
    o_spp, o_pp, o_kinds, o_xy = pack_geometries(orig)
    d_spp, d_pp, d_kinds, d_xy = pack_geometries(dest)
    d_xy = _dest_into_orig(d_xy, pair)
    n_orig, n_dest = len(o_spp) - 1, len(d_spp) - 1
    lib = _lib.load()
    h = C.c_void_p()
    device = current_device() if device is None else device
    _lib.check(lib.atl_intersects_compute(device, n_orig, _lib.ptr(o_spp), _lib.ptr(o_pp), _lib.ptr(o_kinds),
                                          _lib.ptr(o_xy), n_dest, _lib.ptr(d_spp), _lib.ptr(d_pp),
                                          _lib.ptr(d_kinds), _lib.ptr(d_xy), C.byref(h)))
    return _export_csr(lib, h, n_dest, n_orig)


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
    shape_availability_reprojected,
)
from .geotiff import read as read_raster  # noqa: E402


# ---------------------------------------------------------------- regrid (gis.py:765-871 of the reference)

RESAMPLING_NEAREST, RESAMPLING_AVERAGE = 0, 5  # rasterio.enums.Resampling values
# the statistics over the average's boxes (DESIGN.md section 1): rasterio's mode, max, min, med, q1,
# q3, sum and rms
RESAMPLING_STATS = {6: "mode", 8: "max", 9: "min", 10: "med", 11: "q1", 12: "q3", 13: "sum", 14: "rms"}


def _resampling_code(resampling):
    """The int code of ``resampling`` (an int or an enum with an int ``.value``), or
    NotImplementedError for one this package does not offer."""
    code = getattr(resampling, "value", resampling)
    if isinstance(code, bool) or not isinstance(code, (int, np.integer)) or \
            int(code) not in (RESAMPLING_NEAREST, RESAMPLING_AVERAGE, *RESAMPLING_STATS):
        stats = ", ".join(f"{k} ({v})" for k, v in RESAMPLING_STATS.items())
        raise NotImplementedError(f"resampling {resampling!r} is not supported; use 0 (nearest) or 5 (average), "
                                  f"or one of the statistics {stats}")
    return int(code)
REGRID_EPS = 1e-10  # overlaps shorter than this (in source pixels) do not count as overlaps


def _coord(ds, name):
    if name is None:
        raise ValueError("dimx and dimy must carry a .name naming the x / y dimension of the data")
    try:
        return np.asarray(ds.coords[name])
    except KeyError:
        raise ValueError(f"{name!r} names no coordinate of the data") from None


def _spatial_swaps(ds, namex, namey):
    """{dim: slice(None, None, -1)} for the spatial dims whose coordinate descends."""
    swaps = {}
    for name in (namex, namey):
        c = _coord(ds, name)
        if c[-1] < c[0]:
            swaps[name] = slice(None, None, -1)
    return swaps


def maybe_swap_spatial_dims(ds, namex="x", namey="y"):
    """``ds`` with its ``namex`` / ``namey`` axes reversed where their coordinates descend, so both
    ascend (gis.py:765-778).  Works on xarray objects and this package's ``DataArray``; for its
    ``Dataset`` the flipped variables are NumPy views or flipped copies of torch tensors."""
    from .labelled import Dataset, LazyDataset

    swaps = _spatial_swaps(ds, namex, namey)
    if not swaps:
        return ds
    if not isinstance(ds, Dataset):
        return ds.isel(**swaps)
    coords = {k: (np.asarray(v)[::-1] if k in swaps else v) for k, v in ds.coords.items()}

    def flip(arr, dims):
        axes = [dims.index(d) for d in swaps if d in dims]
        if not axes:
            return arr
        return arr.flip(axes) if not isinstance(arr, np.ndarray) else np.flip(arr, axes)

    if isinstance(ds, LazyDataset):
        dims = ("time", "y", "x")
        out = LazyDataset({n: (lambda lo, hi, ld=ld: flip(np.asarray(ld(lo, hi)), dims)) for n, ld in ds._loaders.items()},
                          coords, attrs=ds.attrs, time_chunk=ds.time_chunk, dtypes=ds._dtypes)
    else:
        out = Dataset(coords=coords, attrs=ds.attrs)
    for name, (dims, arr) in ds._vars.items():
        out._vars[name] = (dims, flip(arr, dims))
    return out


def _transform_axis(c, name):
    """(first centre, step) of an evenly spaced axis in its given order, as the reference's
    ``_as_transform`` takes them (gis.py:781-788); descending axes get a negative step.  The
    spacing is checked by ``regular_axis`` on the ascending order."""
    c = np.asarray(c, dtype=np.float64)
    regular_axis(c[::-1] if c.ndim == 1 and len(c) > 1 and c[-1] < c[0] else c, name)
    return float(c[0]), float(c[-1] - c[0]) / float(len(c) - 1)


def regrid_axis(src0, sstep, n_src, dst0, dstep, n_dst, pad, nearest=False):
    """One axis of ``regrid``'s separable weights: (first, count, weights) per destination index,
    over the ascending source axis with centres ``src0 + k * sstep`` (``sstep > 0``), extended by
    ``pad`` pixels on each side that repeat the border pixel.  A destination cell is
    ``[o + j * dstep, o + (j + 1) * dstep]`` with ``o = dst0 - dstep / 2`` (the affine transform).

    average: the overlap length of each source pixel with the cell, in source pixels (pixels whose
    overlap is below ``REGRID_EPS`` are left out); padded pixels add into the border pixel.
    nearest: weight 1 for the pixel that contains the cell centre (a centre on a border takes
    the pixel above it); count 0 when the centre lies outside the padded source."""
    so = src0 - sstep / 2
    do = dst0 - dstep / 2
    first = np.zeros(n_dst, dtype=np.int32)
    count = np.zeros(n_dst, dtype=np.int32)
    weights = []
    for j in range(n_dst):
        if nearest:
            k = math.floor(((do + (j + 0.5) * dstep) - so) / sstep)
            w = {min(max(k, 0), n_src - 1): 1.0} if -pad <= k < n_src + pad else {}
        else:
            e0, e1 = do + j * dstep, do + (j + 1) * dstep
            u0, u1 = (min(e0, e1) - so) / sstep, (max(e0, e1) - so) / sstep
            w = {}
            for k in range(max(math.floor(u0 + REGRID_EPS), -pad), min(math.ceil(u1 - REGRID_EPS), n_src + pad)):
                real = min(max(k, 0), n_src - 1)
                w[real] = w.get(real, 0.0) + (min(k + 1.0, u1) - max(float(k), u0))
        if w:
            first[j], count[j] = min(w), len(w)
        weights.append([w[k] for k in sorted(w)])
    table = np.zeros((n_dst, max([1] + [len(w) for w in weights])), dtype=np.float64)
    for j, w in enumerate(weights):
        table[j, :len(w)] = w
    return first, count, table


def _flip_axis_table(tab, n_src):
    """A table over the ascending axis -> the same over the stored (descending) order."""
    first, count, w = tab
    w = w.copy()
    for j, c in enumerate(count):
        w[j, :c] = w[j, :c][::-1].copy()
    return np.where(count > 0, n_src - first - count, 0).astype(np.int32), count, w


def _crs_key(crs):
    from . import proj

    try:
        return ("epsg", proj.epsg(crs))
    except NotImplementedError:
        return crs


def regrid_op(xs, ys, dimx, dimy, resampling, device):
    """``engine.RegridOp`` from the source centres ``xs`` / ``ys`` (as stored, either order) onto the
    destination centres ``dimx`` / ``dimy`` (their ``.name`` name the dims), with ``regrid``'s tables."""
    from .engine import RegridOp, ReprojectOp

    namex, namey = getattr(dimx, "name", None), getattr(dimy, "name", None)
    swapx, swapy = len(xs) > 1 and xs[-1] < xs[0], len(ys) > 1 and ys[-1] < ys[0]
    # grids as the reference builds them: the source ascending, the destination in its given order
    xs, ys = (xs[::-1] if swapx else xs), (ys[::-1] if swapy else ys)
    sx0, sdx = regular_axis(xs, namex)
    sy0, sdy = regular_axis(ys, namey)
    dx0, ddx = _transform_axis(dimx, namex)
    dy0, ddy = _transform_axis(dimy, namey)
    pad = int(abs(ddx) // min(sdx, sdy) * 1.1)
    nearest = resampling == RESAMPLING_NEAREST
    ytab = regrid_axis(sy0, sdy, len(ys), dy0, ddy, len(dimy), pad, nearest)
    xtab = regrid_axis(sx0, sdx, len(xs), dx0, ddx, len(dimx), pad, nearest)
    if swapy:
        ytab = _flip_axis_table(ytab, len(ys))
    if swapx:
        xtab = _flip_axis_table(xtab, len(xs))
    if resampling in RESAMPLING_STATS:  # the statistics over the average's (padded) boxes
        return ReprojectOp.tables((len(ys), len(xs)), ytab, xtab, resampling, device=device)
    return RegridOp((len(ys), len(xs)), ytab, xtab, device=device)


def regrid(ds, dimx, dimy, **kwargs):
    """Resample ``ds`` onto the regular grid with x centres ``dimx`` and y centres ``dimy``, whose
    ``.name`` name the x and y dims of ``ds`` (gis.py:791-871; a ``pd.Index`` or an xarray
    coordinate).  Only ``resampling`` (0 nearest, the default, 5 average, or a statistic of
    ``RESAMPLING_STATS`` over the average's padded boxes; an int or an enum with an int ``.value``),
    ``src_crs`` and ``dst_crs`` (default 4326, and they must name the same CRS)
    are accepted.

    ``ds``: this package's ``DataArray`` / ``Dataset`` / ``LazyDataset`` or an xarray object; xarray
    in gives xarray out.  Every variable needs both dims; its other dims come first in their order,
    then y, x.  All variables share one dtype, float32 or float64, which the result keeps.  CUDA
    tensors are resampled on their device and stay there; host values give host values; a
    ``LazyDataset`` is resampled one time part at a time.  The result's coordinates along the two
    dims are ``dimy`` / ``dimx`` in the order given, and attrs are kept.  Semantics and deviations
    from GDAL: DESIGN.md section 1."""
    from .engine import _is_torch, current_device
    from .labelled import HAVE_XARRAY, DataArray, Dataset, LazyDataset, xr

    unknown = sorted(set(kwargs) - {"resampling", "src_crs", "dst_crs"})
    if unknown:
        raise TypeError(f"regrid got unsupported keyword argument(s) {unknown}; "
                        "supported are resampling, src_crs and dst_crs")
    code = _resampling_code(kwargs.get("resampling", RESAMPLING_NEAREST))
    src_crs, dst_crs = kwargs.get("src_crs", 4326), kwargs.get("dst_crs", 4326)
    if _crs_key(src_crs) != _crs_key(dst_crs):
        raise NotImplementedError(f"regrid only resamples within one CRS, not from {src_crs!r} to {dst_crs!r}")

    namex, namey = getattr(dimx, "name", None), getattr(dimy, "name", None)
    xs, ys = _coord(ds, namex), _coord(ds, namey)
    is_xr = HAVE_XARRAY and isinstance(ds, (xr.DataArray, xr.Dataset))
    if is_xr:
        items = [(n, tuple(da.dims), da.data) for n, da in
                 (ds.data_vars.items() if isinstance(ds, xr.Dataset) else [(ds.name, ds)])]
    elif isinstance(ds, DataArray):
        items = [(ds.name, ds.dims, ds.values)]
    elif isinstance(ds, Dataset):
        items = [(n, ds.dims_of(n), None if n in getattr(ds, "_loaders", ()) else ds.raw(n)) for n in ds.keys()]
    else:
        raise TypeError(f"regrid takes a DataArray or Dataset, not {type(ds).__name__}")

    def dtype_of(n, arr):
        if arr is None:
            return ds.dtype_of(n)
        return np.dtype(str(arr.dtype).replace("torch.", "")) if _is_torch(arr) else np.dtype(arr.dtype)

    dtypes = {dtype_of(n, a) for n, _, a in items}
    assert len(dtypes) == 1, "regrid can only reproject datasets with homogeneous dtype"
    dtype = dtypes.pop()
    if dtype not in (np.float32, np.float64):
        raise TypeError(f"regrid supports float32 and float64 values, not {dtype}")
    for n, dims, _ in items:
        if namex not in dims or namey not in dims:
            raise ValueError(f"variable {n!r} with dims {dims} lacks the dim {namex!r} or {namey!r}")

    devices = {a.device.index for _, _, a in items if _is_torch(a) and a.is_cuda}
    if len(devices) > 1:
        raise ValueError("the variables of one regrid call live on different GPUs")
    op = regrid_op(xs, ys, dimx, dimy, int(code), devices.pop() if devices else current_device())

    def resample(dims, arr):
        lead = [d for d in dims if d not in (namey, namex)]
        perm = [dims.index(d) for d in lead] + [dims.index(namey), dims.index(namex)]
        if _is_torch(arr):
            if not arr.is_cuda:
                arr = arr.numpy()
            elif arr.shape[dims.index(namex)] > len(xs) and dims[-1] == namex:  # a row-padded device cutout
                arr = arr[..., :len(xs)]
        if arr.shape[dims.index(namey)] != len(ys) or arr.shape[dims.index(namex)] != len(xs):
            raise ValueError(f"values of shape {tuple(arr.shape)} do not match the {namey!r} / {namex!r} coordinates")
        arr = arr.permute(perm) if _is_torch(arr) else np.transpose(arr, perm)
        shape = tuple(arr.shape[:-2])
        res = op(arr.reshape((-1, len(ys), len(xs))))
        return tuple(lead) + (namey, namex), res.reshape(shape + op.dst_shape)

    out_vars = {}
    for n, dims, arr in items:
        if arr is not None:
            out_vars[n] = resample(dims, arr)
    if isinstance(ds, LazyDataset):
        lazy = [n for n, _, arr in items if arr is None]
        nt, parts = len(ds.coords["time"]), {n: [] for n in lazy}
        for lo in range(0, nt, ds.time_chunk):
            part = ds.isel_time(lo, min(nt, lo + ds.time_chunk))
            for n in lazy:
                new_dims, res = resample(part.dims_of(n), part.raw(n))
                parts[n].append(res)
        for n in lazy:
            out_vars[n] = (new_dims, np.concatenate(parts[n]) if parts[n] else
                           np.empty((0,) + op.dst_shape, dtype=dtype))
        out_vars = {n: out_vars[n] for n in ds.keys()}

    newx, newy = np.asarray(dimx), np.asarray(dimy)
    if is_xr:
        def wrap(n, da, dims, values):
            coords = {k: v for k, v in da.coords.items() if namex not in v.dims and namey not in v.dims}
            coords[namey] = (namey, newy, ds.coords[namey].attrs)
            coords[namex] = (namex, newx, ds.coords[namex].attrs)
            values = values.cpu().numpy() if _is_torch(values) else values
            return xr.DataArray(values, coords=coords, dims=dims, name=da.name, attrs=da.attrs)

        if isinstance(ds, xr.Dataset):
            return xr.Dataset({n: wrap(n, ds[n], *out_vars[n]) for n in out_vars}, attrs=ds.attrs)
        return wrap(ds.name, ds, *out_vars[ds.name])
    if isinstance(ds, DataArray):
        dims, values = out_vars[ds.name]
        coords = {k: v for k, v in ds.coords.items() if k in dims and k not in (namex, namey)}
        coords.update({namey: newy, namex: newx})
        return DataArray(values, coords, dims, ds.name, ds.attrs)
    coords = dict(ds.coords)
    for name, new in ((namex, newx), (namey, newy)):
        aliases = next((a for a in Dataset._AXIS_COORDS.values() if name in a), (name,))
        for a in set(aliases) | {name}:
            if a in coords or a == name:
                coords[a] = new
    out = Dataset(coords=coords, attrs=ds.attrs)
    for n, (dims, values) in out_vars.items():
        out._vars[n] = (dims, values)
    return out


# ---------------------------------------------------------------- reproject (rasterio.warp.reproject)

def _axis_transform(t, what):
    """(a, c, e, f) of an axis-aligned affine transform (6-tuple or ``Affine``: x = a col + c,
    y = e row + f); ValueError for a rotated, degenerate or non-finite one."""
    from .availability import _coeffs

    a, b, c, d, e, f = _coeffs(t)
    if b != 0.0 or d != 0.0 or a == 0.0 or e == 0.0 or not np.isfinite([a, c, e, f]).all():
        raise ValueError(f"{what} must be axis-aligned (b = d = 0) with finite, non-zero a and e")
    return a, b, c, d, e, f


def _same_nodata(x, y):
    return (x is None and y is None) or (x is not None and y is not None and
                                         (float(x) == float(y) or (np.isnan(x) and np.isnan(y))))


def _same_crs_tables(src_t, src_shape, dst_t, dst_shape, nearest):
    """``regrid_axis(pad=0)`` tables (y, x) of the destination cells over the source pixels, as stored
    (either sign of a and e), both transforms in one CRS."""
    sa, _, sc, _, se, sf = src_t
    da, _, dc, _, de, df = dst_t

    def axis(s0, ss, n, d0, ds, m):
        if ss > 0:
            return regrid_axis(s0 + ss / 2, ss, n, d0 + ds / 2, ds, m, 0, nearest)
        lo = s0 + n * ss  # the low edge of the descending axis
        return _flip_axis_table(regrid_axis(lo - ss / 2, -ss, n, d0 + ds / 2, ds, m, 0, nearest), n)

    return axis(sf, se, src_shape[0], df, de, dst_shape[0]), axis(sc, sa, src_shape[1], dc, da, dst_shape[1])


def reproject(source, dst_transform, dst_crs, dst_shape, *, src_transform=None, src_crs=None, resampling=0,
              src_nodata=None, dst_nodata=None):
    """Warp ``source`` onto the grid ``dst_transform`` / ``dst_shape`` in ``dst_crs`` on the GPU
    (rasterio.warp.reproject with Resampling.nearest or .average for affine-georeferenced rasters).
    Returns ``(destination, dst_transform)``.

    ``source``: a ``Raster`` (its transform, CRS and nodata are used; a keyword that contradicts them
    raises ``ValueError``) or an array with ``src_transform`` and ``src_crs``: NumPy or a CUDA tensor,
    (ny, nx) or (..., ny, nx), the leading dims a batch that shares the geometry.  float32 or float64,
    kept in the result; a CUDA tensor gives a tensor on its device, NumPy gives NumPy.  A host array
    goes to the device in batch slabs, so one 2-D entry of it must fit in device memory.

    CRSs: any of ``proj.SUPPORTED`` (``proj.epsg``).  Transforms: 6-tuples or ``Affine``, axis-aligned
    (b = d = 0), either sign of a and e, so ``dst_transform=cutout.transform, dst_crs=cutout.crs,
    dst_shape=cutout.shape`` gives rows in the cutout's ascending-y order.  ``resampling``: 0 (nearest),
    5 (average) or a statistic of ``RESAMPLING_STATS`` (sum, rms, min, max, med, q1, q3, mode over the
    average's boxes), an int or an enum with ``.value``.  NaN and ``src_nodata`` are skipped; a cell
    without a valid pixel gets ``dst_nodata`` (default ``src_nodata``, else NaN).  Every argument is
    checked before any device work.  Within one CRS the footprints are separable and the call runs
    ``regrid``'s kernel on ``regrid_axis(pad=0)`` tables, unless a cell spans more source columns than
    that kernel's shared memory holds (``RegridOp.ring_fits``); then, and across CRSs, it runs
    atl_reproject.  The statistics run atl_reproject_ex, on those tables where the average would run
    ``regrid``'s kernel.  Semantics
    and deviations from GDAL: DESIGN.md section 1."""
    from . import proj
    from .engine import RegridOp, ReprojectOp, _is_torch, current_device

    if isinstance(source, Raster):
        own = {"src_transform": tuple(source.transform), "src_crs": source.crs, "src_nodata": source.nodata}
        given = {"src_transform": src_transform, "src_crs": src_crs, "src_nodata": src_nodata}
        for k, v in given.items():
            if v is None:
                continue
            same = (_axis_transform(v, k) == own[k] if k == "src_transform" else
                    proj.epsg(v) == proj.epsg(own[k]) if k == "src_crs" else _same_nodata(v, own[k]))
            if not same:
                raise ValueError(f"{k}={v!r} contradicts the raster's {own[k]!r}")
        arr, src_transform, src_crs, src_nodata = source.array, own["src_transform"], source.crs, source.nodata
    else:
        arr = source
        if src_transform is None or src_crs is None:
            raise ValueError("an array source needs src_transform and src_crs")
    code = _resampling_code(resampling)
    skey, dkey = proj.epsg(src_crs), proj.epsg(dst_crs)
    st = _axis_transform(src_transform, "src_transform")
    dt = _axis_transform(dst_transform, "dst_transform")
    try:
        dst_shape = tuple(int(n) for n in dst_shape)
    except TypeError:
        raise ValueError(f"dst_shape must be (ny, nx), not {dst_shape!r}") from None
    if len(dst_shape) != 2 or min(dst_shape) < 0:
        raise ValueError(f"dst_shape must be two non-negative sizes (ny, nx), not {dst_shape!r}")
    for name, v in (("src_nodata", src_nodata), ("dst_nodata", dst_nodata)):
        if v is not None and not isinstance(v, (int, float, np.integer, np.floating)) or isinstance(v, bool):
            raise TypeError(f"{name} must be a number or None, not {v!r}")
    if not hasattr(arr, "ndim") or not hasattr(arr, "shape"):
        arr = np.asarray(arr)
    on_device = _is_torch(arr) and arr.is_cuda
    if _is_torch(arr) and not on_device:
        arr = arr.numpy()
    dtype = np.dtype(str(arr.dtype).replace("torch.", ""))
    if dtype not in (np.float32, np.float64):
        raise TypeError(f"reproject supports float32 and float64 values, not {dtype}")
    if arr.ndim < 2 or min(arr.shape[-2:]) < 1:
        raise ValueError(f"the source must be (..., ny, nx) with ny, nx >= 1, not of shape {tuple(arr.shape)}")
    dst_nodata = (src_nodata if src_nodata is not None else np.nan) if dst_nodata is None else dst_nodata

    lead, src_shape = tuple(arr.shape[:-2]), tuple(int(n) for n in arr.shape[-2:])
    flat = arr.reshape((-1,) + src_shape)
    device = arr.device.index if on_device else current_device()
    nearest = code == RESAMPLING_NEAREST
    tables = _same_crs_tables(st, src_shape, dt, dst_shape, nearest) if skey == dkey else None
    if tables is not None and RegridOp.ring_fits(tables[1]):
        if code in RESAMPLING_STATS:  # the statistics over the average's boxes
            out = ReprojectOp.tables(src_shape, *tables, code, src_nodata, dst_nodata, device)(flat)
        else:
            out = RegridOp(src_shape, *tables, device=device)(flat, nodata=src_nodata, empty=dst_nodata)
    else:  # across CRSs, or (on the identity pair) a cell wider than k_regrid's shared-memory row ring
        op = ReprojectOp((st, src_shape, skey), (dt, dst_shape, dkey), code, src_nodata, dst_nodata, device)
        out = op(flat)
    return out.reshape(lead + dst_shape), dst_transform
