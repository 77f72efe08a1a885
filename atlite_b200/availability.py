"""Land eligibility: ``ExclusionContainer``, ``shape_availability`` and the availability matrix
(the reference's gis.py:186-325 and 376-583, cutout.py:517 ``availabilitymatrix``).

Per shape, on a window of ``res``-sized pixels in the container's CRS (``padded_transform_and_shape``
of the projected shape's bounds):

1. pixels whose centre is outside the shape are excluded (even-odd rule, exact orientation signs);
2. every raster excludes the pixels whose nearest raster pixel is excluded by its ``codes`` rule
   (``nodata`` outside the raster, outside the shape and where the raster holds it), ``invert``-ed,
   then dilated ``int(buffer / res) + 1`` times with the 4-connected cross;
3. every geometry collection excludes the centres inside it or within ``buffer`` of it (a negative
   buffer on a polygon: the centres deeper than ``|buffer|`` inside), ``invert``-ed;
4. the eligible pixels are counted per cutout cell by their centre, and
   ``A = count * res^2 / area(cell)``;
5. or, with ``compute_shape_availability(dst_transform=, dst_crs=, dst_shape=)``, the mask is padded
   with ineligible pixels and averaged over each destination cell's footprint (``gis.reproject``'s
   average, from nine exact counts per cell).

Every stage runs in csrc/availability.cu; polygon vertices are projected here (``proj``), pixel
centres on the device.  A window larger than ``_Session.BAND_BYTES`` (or than free device memory)
is processed in bands of whole rows, each with the halo of rows its raster buffers need, so any
window runs; only the host result of ``shape_availability`` must fit host memory.  Rasters are ``Raster`` objects, GeoTIFF paths (read onto the device by
``geotiff.read``), or rasterio datasets / other paths when rasterio is installed, and are uploaded
once per call.
"""

from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _lib, gis, proj
from .engine import _dptr, _is_torch, _stream_ptr, _torch, current_device


# ---------------------------------------------------------------- lattice helpers
def padded_transform_and_shape(bounds, res):
    """(transform, (ny, nx)) of the ``res`` raster around ``bounds`` = (left, bottom, right, top),
    with the reference's float64 arithmetic (gis.py:186-194).  The transform is the 6-tuple
    (res, 0, left, 0, -res, top) (a ``rasterio.Affine`` when rasterio is installed)."""
    from .cutout import _affine

    left, bottom = ((float(b) // res) * res for b in bounds[:2])
    right, top = ((float(b) // res + 1) * res for b in bounds[2:])
    shape = int((top - bottom) / res), int((right - left) / res)
    return _affine(res, 0, left, 0, -res, top), shape


def _coeffs(transform):
    t = tuple(float(v) for v in list(transform)[:6])
    if len(t) != 6:
        raise ValueError("a transform needs the six affine coefficients (a, b, c, d, e, f)")
    return t


class Raster:
    """An in-memory raster: ``array`` (2-D NumPy array or CUDA tensor, integer, bool or float),
    ``transform`` (a 6-tuple (a, b, c, d, e, f) or an ``Affine``: x = a col + c, y = e row + f; north
    up, so b = d = 0, a > 0 and e < 0), ``crs`` (one of ``proj.SUPPORTED``) and ``nodata`` (the file's
    nodata value, or None; informative only: ``add_raster(nodata=)`` decides what is nodata)."""

    def __init__(self, array, transform, crs, nodata=None):
        if array.ndim != 2:
            raise ValueError("a raster must be 2-D")
        a, b, c, d, e, f = _coeffs(transform)
        if b != 0.0 or d != 0.0 or not a > 0.0 or not e < 0.0:
            raise ValueError("only north-up rasters are supported (transform b = d = 0, a > 0, e < 0)")
        self.array = array
        self.transform = (a, b, c, d, e, f)
        self.crs = crs
        self.epsg = proj.epsg(crs)
        self.nodata = nodata

    @property
    def shape(self):
        return tuple(int(s) for s in self.array.shape)

    @property
    def bounds(self):
        """(left, bottom, right, top)."""
        a, _, c, _, e, f = self.transform
        ny, nx = self.shape
        return c, f + ny * e, c + nx * a, f

    def __repr__(self):
        return f"<Raster {self.shape[1]} x {self.shape[0]} {proj.name(self.epsg)}>"


def _is_path(obj):
    return isinstance(obj, (str, os.PathLike))


# ---------------------------------------------------------------- container
class ExclusionContainer:
    """Rasters and geometries to exclude, on a ``res`` lattice in ``crs`` (gis.py:376-583)."""

    def __init__(self, crs=3035, res=100):
        self.rasters = []
        self.geometries = []
        self.crs = crs
        self.res = res
        proj.epsg(crs)

    def add_raster(self, raster, codes=None, buffer=0, invert=False, nodata=255, allow_no_overlap=False, crs=None):
        """Register a raster: a ``Raster``, a GeoTIFF path, a rasterio dataset or another path
        (rasterio needed; see ``open_files``).  ``codes``:
        None (every non-zero value is excluded), a value or list of values, or an elementwise callable
        (evaluated once on the raster's distinct values).  ``buffer`` in units of the container's CRS.
        ``crs``: the raster's CRS when the dataset has none."""
        self.rasters.append(dict(raster=raster, codes=codes, buffer=buffer, invert=invert, nodata=nodata,
                                 allow_no_overlap=allow_no_overlap, crs=crs))

    def add_geometry(self, geometry, buffer=0, invert=False):
        """Register a collection of geometries (any form ``gis.geometry_parts`` reads, a GeoSeries /
        GeoDataFrame, or a path geopandas reads).  Its CRS is its ``.crs``, else the container's."""
        self.geometries.append(dict(geometry=geometry, buffer=buffer, invert=invert))

    def open_files(self):
        """Read the rasters given as rasterio datasets or paths (band 1) and the geometries given as
        paths.  A path to a GeoTIFF that ``geotiff.read`` supports is read by it onto the current
        device when its GeoKeys name an EPSG code, or when rasterio is not installed and ``crs`` was
        given; every other path is opened with rasterio."""
        from . import geotiff

        try:
            import rasterio  # noqa: F401

            have_rasterio = True
        except ImportError:
            have_rasterio = False
        for d in self.rasters:
            r = d["raster"]
            if isinstance(r, Raster):
                continue
            if _is_path(r) and geotiff.readable(r, None if have_rasterio else d["crs"]):
                d["raster"] = geotiff.read(r, crs=d["crs"], device=current_device())
                continue
            try:
                import rasterio
            except ImportError as e:
                raise ImportError(f"reading the raster {r!r} needs rasterio, which is not installed; "
                                  "pass a gis.Raster(array, transform, crs) instead") from e
            if _is_path(r):
                r = rasterio.open(r)
            crs = r.crs if r.crs is not None else d["crs"]
            if crs is None:
                raise ValueError(f"CRS of {r} is undefined, please provide it manually (crs=)")
            d["raster"] = Raster(r.read(1), r.transform, crs)
        for d in self.geometries:
            g = d["geometry"]
            if _is_path(g):
                try:
                    import geopandas as gpd
                except ImportError as e:
                    raise ImportError(f"reading the geometries {g!r} needs geopandas, which is not installed; "
                                      "pass the geometries themselves instead") from e
                g = gpd.read_file(g)
            if hasattr(g, "columns") and hasattr(g, "geometry"):
                g = g.geometry
            d["geometry"] = g

    @property
    def all_closed(self):
        return all(_is_path(d["raster"]) for d in self.rasters) and all(_is_path(d["geometry"])
                                                                       for d in self.geometries)

    @property
    def all_open(self):
        return all(isinstance(d["raster"], Raster) for d in self.rasters) and not any(
            _is_path(d["geometry"]) for d in self.geometries)

    def __repr__(self):
        return (f"Exclusion Container"
                f"\n registered rasters: {len(self.rasters)} "
                f"\n registered geometry collections: {len(self.geometries)}"
                f"\n CRS: {self.crs} - Resolution: {self.res}")

    def compute_shape_availability(self, geometry, dst_transform=None, dst_crs=None, dst_shape=None, crs=None):
        """(eligible mask, transform) of ``geometry`` (one shape or a collection, combined), projected to
        the container's CRS first.  ``crs``: the geometry's CRS when it has no ``.crs`` (default: the
        container's).

        With ``dst_transform``, ``dst_crs`` and ``dst_shape`` (all three, or none): ``(values,
        dst_transform)``, ``values`` the float64 (ny, nx) eligible share of each cell of that grid, the
        mask averaged over each cell's footprint after padding it with ineligible pixels (the
        reference's ``shape_availability_reprojected``; semantics in DESIGN.md section 1).  Any CRS of
        ``proj.SUPPORTED``; the transform axis-aligned with either sign of a and e, so
        ``cutout.transform`` and ``cutout.transform_r`` both work."""
        given = [v is not None for v in (dst_transform, dst_crs, dst_shape)]
        if any(given) and not all(given):
            raise NotImplementedError("dst_transform, dst_crs and dst_shape must be given together to reproject the "
                                      "availability; for the availability aggregated to a cutout's cells see also "
                                      "Cutout.availabilitymatrix")
        src = _crs_of(geometry, crs, self.crs)
        dst = _dst_lattice(dst_transform, dst_crs, dst_shape) if all(given) else None
        with _Session(self) as s:
            parts = _parts(geometry, src, proj.epsg(self.crs), polygonal=True)
            if dst is None:
                return s.shape_mask(parts)
            return s.average(parts, dst, dst_crs), dst_transform


def shape_availability(geometry, excluder, crs=None):
    """(eligible mask as a NumPy bool (ny, nx) array, row 0 at the top, and its transform) of
    ``geometry`` (gis.py:263-325).  The geometry must be in the container's CRS (its ``.crs``, else
    ``crs``, else the container's own is assumed)."""
    src = _crs_of(geometry, crs, excluder.crs)
    if proj.epsg(src) != proj.epsg(excluder.crs):
        raise ValueError(f"the geometry's CRS ({src}) differs from the exclusion container's ({excluder.crs}); "
                         "project it first or use ExclusionContainer.compute_shape_availability")
    with _Session(excluder) as s:
        return s.shape_mask(_parts(geometry, src, proj.epsg(excluder.crs), polygonal=True))


def shape_availability_reprojected(geometry, excluder, dst_transform, dst_crs, dst_shape, crs=None):
    """(values, dst_transform): the eligible share of each cell of the grid ``dst_transform`` /
    ``dst_crs`` / ``dst_shape`` (gis.py:328-373), as ``excluder.compute_shape_availability`` with the
    three ``dst_*`` arguments."""
    if any(v is None for v in (dst_transform, dst_crs, dst_shape)):
        raise ValueError("shape_availability_reprojected needs dst_transform, dst_crs and dst_shape")
    return excluder.compute_shape_availability(geometry, dst_transform, dst_crs, dst_shape, crs=crs)


def _dst_lattice(dst_transform, dst_crs, dst_shape):
    """The checked destination grid of a reprojected availability as a ``_lib.Lattice``."""
    proj.epsg(dst_crs)
    a, _, c, _, e, f = gis._axis_transform(dst_transform, "dst_transform")
    shape = tuple(dst_shape) if isinstance(dst_shape, (tuple, list)) else None
    if (shape is None or len(shape) != 2 or
            not all(isinstance(n, (int, np.integer)) and not isinstance(n, bool) and n > 0 for n in shape)):
        raise ValueError(f"dst_shape must be two positive ints (ny, nx), not {dst_shape!r}")
    if max(shape) >= 2 ** 31 - 1:
        raise ValueError(f"dst_shape {dst_shape!r} is too large")
    return _lattice(c, a, f, e, shape[1], shape[0])


def reprojection_pad(transform, crs, dst_a, dst_crs):
    """Pixels of value 0 added around a window before its reprojected average (the reference's
    ``pad_extent``, gis.py:233-260): ``int(dst_a // covered_res * 1.1)``, ``covered_res`` the smaller
    side of the bounds in ``dst_crs`` of the window's first pixel T (0, 0) .. T (1, 1), taken as
    rasterio's ``transform_bounds`` does (each edge densified with 21 points).  Points without an image
    are left out; 0 for a negative ``dst_a``."""
    a, _, c, _, e, f = _coeffs(transform)
    left, top, right, bottom = c, f, c + a, f + e
    t = np.linspace(0.0, 1.0, 23)  # the corners and 21 points between them
    xs = np.r_[left + (right - left) * t, np.full_like(t, right), right + (left - right) * t, np.full_like(t, left)]
    ys = np.r_[np.full_like(t, bottom), bottom + (top - bottom) * t, np.full_like(t, top), top + (bottom - top) * t]
    px, py = proj.transform(xs, ys, crs, dst_crs)
    ok = np.isfinite(px) & np.isfinite(py)
    if not ok.any():
        raise ValueError(f"the window's first pixel has no image in {proj.name(dst_crs)}")
    covered_res = min(abs(float(px[ok].max() - px[ok].min())), abs(float(py[ok].max() - py[ok].min())))
    if not covered_res > 0.0:
        raise ValueError(f"the window's first pixel has no extent in {proj.name(dst_crs)}")
    return max(int(float(dst_a) // covered_res * 1.1), 0)


def compute_availabilitymatrix(cutout, shapes, excluder, nprocesses=None, disable_progressbar=True, shapes_crs=None):
    """(shape, y, x) float64 share of each cutout cell that is eligible and inside each shape
    (gis.py:586-661).  Shapes take their CRS from ``.crs``, else ``shapes_crs``, else the cutout's.
    ``nprocesses`` and ``disable_progressbar`` are accepted and unused: the shapes run one after
    another on the GPU."""
    from .labelled import make_dataarray

    x = np.asarray(cutout.coords["x"], dtype=np.float64)
    y = np.asarray(cutout.coords["y"], dtype=np.float64)
    cont, cut = proj.epsg(excluder.crs), proj.epsg(cutout.crs)
    if cont != cut and cut != 4326:
        raise NotImplementedError(f"a {proj.name(cut)} cutout needs a {proj.name(cut)} exclusion container")
    src = _crs_of(shapes, shapes_crs, cutout.crs)
    geoms = gis._iter_shapes(shapes)
    import pandas as pd

    index = getattr(shapes, "index", None)
    if not isinstance(index, pd.Index):  # a list's .index is a method
        index = pd.RangeIndex(len(geoms))
    dim = index.name if index.name is not None else "dim_0"
    dx, dy = cutout.dx, cutout.dy
    with _Session(excluder) as s:
        counts = s.counts([_parts(g, src, cont, polygonal=True) for g in geoms],
                          (x[0] - dx / 2, dx, y[0] - dy / 2, dy, len(x), len(y)), cut)
    res = float(excluder.res)
    if cont == cut:
        area = np.full((len(y), len(x)), abs(dx * dy))
    else:
        xlo = x[0] - dx / 2 + np.arange(len(x)) * dx
        ylo = y[0] - dy / 2 + np.arange(len(y)) * dy
        area = proj.cell_area(cont, xlo[None, :], xlo[None, :] + dx, ylo[:, None], ylo[:, None] + dy)
    A = counts.astype(np.float64) * (res * res) / area
    return make_dataarray(A, (dim, "y", "x"), {dim: np.asarray(index), "y": y, "x": x})


# ---------------------------------------------------------------- geometry packing
def _crs_of(obj, crs, default):
    c = getattr(obj, "crs", None)
    return c if c is not None else (crs if crs is not None else default)


class _Parts:
    """The parts of one shape or collection, projected: rings (with hole flags), lines, points."""

    def __init__(self, rings, lines, points):
        self.rings, self.lines, self.points = rings, lines, points

    def bounds(self):
        v = [r for r, _ in self.rings] + self.lines + self.points
        if not v:
            return None
        v = np.concatenate(v)
        return v[:, 0].min(), v[:, 1].min(), v[:, 0].max(), v[:, 1].max()

    def edges(self, orient=False):
        """(n, 4) ring edges (closing edges included) and their weights: 1, or with ``orient`` the
        ring's orientation sign (+1 for a counter-clockwise exterior or clockwise hole)."""
        e, w = [], []
        for r, hole in self.rings:
            nxt = np.roll(r, -1, axis=0)
            e.append(np.c_[r, nxt])
            s = 1
            if orient:
                area = np.dot(r[:, 0] - r[0, 0], nxt[:, 1] - r[0, 1]) - np.dot(nxt[:, 0] - r[0, 0], r[:, 1] - r[0, 1])
                s = 1 if (area > 0) != hole else -1
            w.append(np.full(len(r), s, dtype=np.int32))
        if not e:
            return np.zeros((0, 4)), np.zeros(0, dtype=np.int32)
        return np.ascontiguousarray(np.concatenate(e)), np.concatenate(w)

    def segments(self):
        """(n, 4) segments whose distance a buffer measures: ring edges, line pieces, points."""
        s = [self.edges()[0]] + [np.c_[a[:-1], a[1:]] for a in self.lines if len(a) > 1]
        s += [np.c_[a, a] for a in self.lines if len(a) == 1] + [np.c_[p, p] for p in self.points]
        return np.ascontiguousarray(np.concatenate(s)) if s else np.zeros((0, 4))


def _project(a, src, dst):
    """(n, 2) vertices from CRS ``src`` to ``dst``; ``ValueError`` for a vertex without an image."""
    p = np.stack(proj.transform(a[:, 0], a[:, 1], src, dst), axis=1)
    if not np.isfinite(p).all():
        bad = a[~np.isfinite(p).all(axis=1)][0]
        raise ValueError(f"the vertex ({bad[0]!r}, {bad[1]!r}) in {proj.name(src)} has no image in {proj.name(dst)}")
    return p


def _parts(geometry, src, dst, polygonal):
    """Parts of a shape or a collection of shapes, projected from CRS ``src`` to ``dst``."""
    single = ((isinstance(geometry, dict) and "type" in geometry) or gis._is_ring(geometry)
              or (hasattr(geometry, "__geo_interface__") and not hasattr(geometry, "index"))
              or (isinstance(geometry, (list, tuple)) and len(geometry) > 0 and all(gis._is_ring(r) for r in geometry)))
    geoms = [geometry] if single else gis._iter_shapes(geometry)
    rings, lines, points = [], [], []
    for g in geoms:
        for kind, a in gis.geometry_parts(g, polygonal=polygonal):
            a = _project(a, src, dst)
            if kind in (gis.PART_EXTERIOR, gis.PART_HOLE):
                rings.append((a, kind == gis.PART_HOLE))
            elif kind == gis.PART_LINE:
                lines.append(a)
            else:
                points.append(a)
    return _Parts(rings, lines, points)


def _lattice(c, a, f, e, nx, ny):
    return _lib.Lattice(float(c), float(a), float(f), float(e), int(nx), int(ny))


def _edge_rows(edges, f, e, row0, ny):
    """First row (counted from lattice row ``row0``) and row count per edge: a superset of the rows
    row0 .. row0 + ny - 1 whose centre y = f + (j + 0.5) e lies in [min(y1, y2), max(y1, y2)); the
    kernel tests each row exactly."""
    ylo = np.minimum(edges[:, 1], edges[:, 3])
    yhi = np.maximum(edges[:, 1], edges[:, 3])
    j0 = np.clip(np.floor((yhi - f) / e - 0.5) - row0, 0, ny - 1)
    j1 = np.clip(np.floor((ylo - f) / e - 0.5) + 1 - row0, -1, ny - 1)
    n = np.maximum(j1 - j0 + 1, 0).astype(np.int64)
    return j0.astype(np.int32), n


def _rule(codes, values):
    if callable(codes):
        r = np.asarray(codes(values)).astype(bool)
        if r.shape != values.shape:
            raise ValueError("a callable `codes` must be elementwise (return an array of its argument's shape)")
        return r
    if codes is not None and np.size(codes) > 0 and (np.ndim(codes) > 0 or bool(codes)):
        return np.isin(values, codes)
    return values.astype(bool)


# ---------------------------------------------------------------- the device session
class _Session:
    """One call's device state: every raster uploaded once, as lookup-table indices."""

    def __init__(self, excluder):
        if not excluder.all_open:
            excluder.open_files()
        self.ex = excluder
        self.res = float(excluder.res)
        self.crs = proj.epsg(excluder.crs)
        self.torch = _torch()
        self.device = current_device()
        self.dev = f"cuda:{self.device}"
        self.lib = _lib.load()
        self._uploads = {}
        self.geoms = [self._prepare_geometry(d) for d in excluder.geometries]  # host only: checks first
        self.rasters = [self._prepare_raster(d) for d in excluder.rasters]

    def __enter__(self):
        self._ctx = self.torch.cuda.device(self.device)
        self._ctx.__enter__()
        return self

    def __exit__(self, *a):
        return self._ctx.__exit__(*a)

    # ---- preparation
    def _upload(self, r):
        key = id(r)
        if key in self._uploads:
            return self._uploads[key]
        torch = self.torch
        arr = r.array
        t = arr if _is_torch(arr) else torch.from_numpy(np.ascontiguousarray(arr))
        dtype = t[:0].cpu().numpy().dtype
        t = t.to(self.dev).contiguous()
        if dtype == np.bool_:
            t, dtype = t.to(torch.uint8), np.dtype(np.uint8)
        if dtype.kind in "iu" and dtype.itemsize <= 2:
            info = np.iinfo(dtype)
            values = np.arange(info.min, info.max + 1).astype(dtype)
            idx = t.to(torch.int32) - int(info.min)
            idx, nbytes = (idx.to(torch.uint8), 1) if dtype.itemsize == 1 else (idx, 4)
        else:
            u, inv = torch.unique(t, return_inverse=True)
            values, idx, nbytes = u.cpu().numpy(), inv.to(torch.int32).contiguous(), 4
        up = (idx.contiguous(), nbytes, values, dtype)
        self._uploads[key] = up
        return up

    def _prepare_raster(self, d):
        r = d["raster"]
        idx, nbytes, values, dtype = self._upload(r)
        lut = _rule(d["codes"], values)
        nd = np.asarray(d["nodata"], dtype=np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            ndc = nd.astype(dtype)
        back = ndc.astype(np.float64)
        if not (back == nd or (np.isnan(nd) and np.isnan(back))):
            raise ValueError(f"nodata {d['nodata']!r} is not representable in the raster's dtype {dtype}")
        ex_nodata = bool(_rule(d["codes"], ndc.reshape(1))[0])
        if d["invert"]:
            lut, ex_nodata = ~lut, not ex_nodata
        k = 0
        if d["buffer"]:
            k = int(d["buffer"] / self.res) + 1
            if k < 1:
                raise ValueError(f"a raster buffer must be positive, not {d['buffer']!r}")
        lut_d = self.torch.from_numpy(np.ascontiguousarray(lut, dtype=np.uint8)).to(self.dev)
        return dict(raster=r, idx=idx, nbytes=nbytes, lut=lut_d, ex_nodata=int(ex_nodata), k=k,
                    allow_no_overlap=bool(d["allow_no_overlap"]))

    def _prepare_geometry(self, d):
        buffer = float(d["buffer"] or 0.0)
        p = _parts(d["geometry"], _crs_of(d["geometry"], None, self.ex.crs), self.crs, polygonal=False)
        if (p.lines or p.points) and not buffer > 0:
            raise ValueError("lines and points can only be excluded with a positive buffer (an unbuffered line has "
                             "no interior)")
        edges, w = p.edges(orient=True)
        segs = p.segments() if buffer != 0.0 else np.zeros((0, 4))
        return dict(edges=edges, w=w, segs=segs, buffer=buffer, invert=bool(d["invert"]))

    # ---- per window
    BAND_BYTES = 16 << 30  # device memory for one band of a shape's window, at PIXEL_BYTES per pixel
    PIXEL_BYTES = 11

    def _h2d(self, a, dt):
        return self.torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(self.dev)

    def _mask(self, L, row0, edges, w, out, cnt, mode, flip):
        """Polygon mask of rows row0 .. row0 + L.ny - 1 of the lattice L, from the edges crossing them."""
        if len(edges):
            first, n = _edge_rows(edges, L.f, L.e, row0, L.ny)
            keep = n > 0
            edges, w, first, n = edges[keep], w[keep], first[keep], n[keep]
        if len(edges):
            ptr = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
            e_d, w_d, r_d, p_d = (self._h2d(edges, np.float64), self._h2d(w, np.int32), self._h2d(first, np.int32),
                                  self._h2d(ptr, np.int64))
            args = (len(edges), _dptr(e_d), _dptr(w_d), _dptr(p_d), _dptr(r_d))
        else:
            args = (0, None, None, None, None)
        _lib.check(self.lib.atl_avail_mask(self.device, C.byref(L), int(row0), *args, _dptr(cnt), _dptr(out), mode,
                                           1 if flip else 0, _stream_ptr()))

    def _band_rows(self, nx, ny):
        """Rows per band of an (ny, nx) window, or ny when it is processed in one pass."""
        free = self.torch.cuda.mem_get_info(self.device)[0]
        budget = min(self.BAND_BYTES, free)
        if self.PIXEL_BYTES * nx * ny <= budget:
            return ny
        halo = max([rd["k"] for rd in self.rasters] + [0])
        rows = budget // (self.PIXEL_BYTES * nx) - 2 * halo
        if rows < 1:
            raise MemoryError(f"one band of the availability window ({nx} pixels wide, with {2 * halo} halo rows) "
                              f"needs more than {budget} bytes of device memory; use a coarser resolution")
        return int(rows)

    def bands(self, parts):
        """The window of one shape, band by band: (exclusions of the band's rows, a uint8 device tensor
        with 1 = excluded; the band lattice; its first row; the window's transform and shape).  Each band
        is computed on its rows plus the dilation halo of the rasters' buffers, so every row equals the
        one-pass result."""
        torch = self.torch
        b = parts.bounds()
        if b is None:
            raise ValueError("a shape without polygon parts has no availability window")
        transform, (ny, nx) = padded_transform_and_shape(b, self.res)
        _, _, left, _, _, top = _coeffs(transform)
        rows = self._band_rows(nx, ny)
        halo = max([rd["k"] for rd in self.rasters] + [0]) if rows < ny else 0
        edges, w = parts.edges()
        for j0 in range(0, ny, rows):
            j1 = min(j0 + rows, ny)
            h0, h1 = max(j0 - halo, 0), min(j1 + halo, ny)
            L = _lattice(left, self.res, top, -self.res, nx, h1 - h0)
            excl = torch.empty((h1 - h0, nx), dtype=torch.uint8, device=self.dev)
            cnt = torch.empty((h1 - h0, nx), dtype=torch.int32, device=self.dev)
            scratch = None
            self._mask(L, h0, edges, w, excl, cnt, _lib.MASK_EVEN_ODD, flip=True)
            for rd in self.rasters:
                if scratch is None:
                    scratch = torch.empty((h1 - h0, nx), dtype=torch.uint8, device=self.dev)
                self._raster(L, h0, parts, rd, excl, cnt, scratch, banded=rows < ny)
            for gd in self.geoms:
                if scratch is None:
                    scratch = torch.empty((h1 - h0, nx), dtype=torch.uint8, device=self.dev)
                self._geometry(L, h0, gd, excl, cnt, scratch)
            yield excl[j0 - h0:j1 - h0], _lattice(left, self.res, top, -self.res, nx, j1 - j0), j0, transform, (ny, nx)

    def _reach(self, L, row0, r):
        """Raster rows [lo, hi) that the centres of rows row0 .. row0 + L.ny - 1 of L can fall in (None:
        not bounded here)."""
        a, _, c, _, e, f = r.transform
        x0, x1 = L.c, L.c + L.nx * L.a
        ytop, ybot = L.f + row0 * L.e, L.f + (row0 + L.ny) * L.e
        if r.epsg == self.crs:
            ys = np.array([ytop, ybot])
        else:  # the image of the band's outline bounds the image of the band
            t = np.linspace(0.0, 1.0, 1025)
            bx = np.r_[x0 + (x1 - x0) * t, np.full_like(t, x1), x1 - (x1 - x0) * t, np.full_like(t, x0)]
            by = np.r_[np.full_like(t, ytop), ytop + (ybot - ytop) * t, np.full_like(t, ybot), ybot - (ybot - ytop) * t]
            ys = proj.transform(bx, by, self.crs, r.epsg)[1]
            if not np.isfinite(ys).all():
                return None
        return int(np.floor((ys.max() - f) / e)) - 2, int(np.floor((ys.min() - f) / e)) + 3

    def _raster(self, L, row0, parts, rd, excl, cnt, scratch, banded):
        torch = self.torch
        r = rd["raster"]
        a, _, c, _, e, f = r.transform
        rny, rnx = r.shape
        s = _lib.RasterSample()
        s.win, s.ras, s.win_row0 = L, _lattice(c, a, f, e, rnx, rny), row0
        s.proj = proj.device_projection(self.crs, r.epsg)
        s.idx, s.idx_bytes = rd["idx"].data_ptr(), rd["nbytes"]
        s.lut, s.ex_nodata = rd["lut"].data_ptr(), rd["ex_nodata"]
        rp = parts if r.epsg == self.crs else _Parts([(_project(q, self.crs, r.epsg), h) for q, h in parts.rings], [], [])
        bx0, by0, bx1, by1 = rp.bounds()
        left, bottom, right, top = r.bounds
        overlap = bx0 < right and bx1 > left and by0 < top and by1 > bottom
        mask = None
        if not overlap:
            if not rd["allow_no_overlap"]:
                raise ValueError("Input shapes do not overlap raster.")
        else:
            i0 = max(int(np.floor((bx0 - c) / a)), 0)
            i1 = min(int(np.floor((bx1 - c) / a)) + 1, rnx)
            j0 = max(int(np.floor((by1 - f) / e)), 0)
            j1 = min(int(np.floor((by0 - f) / e)) + 1, rny)
            # the shape's mask on the raster pixels [i0, i1) x [j0, j1), computed only on the rows the
            # band reaches; its lattice is that of the whole range, so every band sees the same centres
            m0, m1 = j0, j1
            reach = self._reach(L, row0, r) if banded else None
            if reach is not None:
                m0, m1 = max(m0, reach[0]), min(m1, reach[1])
            if i1 > i0 and m1 > m0:
                ML = _lattice(c + i0 * a, a, f + j0 * e, e, i1 - i0, m1 - m0)
                mask = torch.empty((m1 - m0, i1 - i0), dtype=torch.uint8, device=self.dev)
                mcnt = torch.empty((m1 - m0, i1 - i0), dtype=torch.int32, device=self.dev)
                self._mask(ML, m0 - j0, *rp.edges(), mask, mcnt, _lib.MASK_EVEN_ODD, flip=False)
                s.mask, s.mask_i0, s.mask_j0, s.mask_nx, s.mask_ny = mask.data_ptr(), i0, m0, i1 - i0, m1 - m0
        k = rd["k"]
        s.out, s.or_into = (scratch if k else excl).data_ptr(), 0 if k else 1
        _lib.check(self.lib.atl_avail_raster_sample(self.device, C.byref(s), _stream_ptr()))
        if k:
            _lib.check(self.lib.atl_avail_dilate(self.device, L.ny, L.nx, k, _dptr(scratch), _dptr(cnt), _dptr(excl),
                                                 _stream_ptr()))

    def _geometry(self, L, row0, gd, excl, cnt, scratch):
        torch = self.torch
        b = abs(gd["buffer"])
        x0, x1 = L.c, L.c + L.nx * L.a
        y1, y0 = L.f + row0 * L.e, L.f + (row0 + L.ny) * L.e
        g = _lib.GeomExclusion()
        g.win, g.buffer, g.invert, g.excl = L, gd["buffer"], int(gd["invert"]), excl.data_ptr()
        ed, w = gd["edges"], gd["w"]
        if len(ed):  # edges that cross the band's rows and reach its left side or beyond
            keep = (np.maximum(ed[:, 1], ed[:, 3]) >= y0) & (np.minimum(ed[:, 1], ed[:, 3]) <= y1) & (
                np.maximum(ed[:, 0], ed[:, 2]) >= x0)
            ed, w = ed[keep], w[keep]
        if len(ed):
            self._mask(L, row0, ed, w, scratch, cnt, _lib.MASK_NONZERO, flip=False)
            g.inside = scratch.data_ptr()
        sg = gd["segs"]
        if len(sg):
            keep = (np.maximum(sg[:, 0], sg[:, 2]) >= x0 - b) & (np.minimum(sg[:, 0], sg[:, 2]) <= x1 + b) & (
                np.maximum(sg[:, 1], sg[:, 3]) >= y0 - b) & (np.minimum(sg[:, 1], sg[:, 3]) <= y1 + b)
            sg = sg[keep]
        if len(sg):  # tensors freed here are only reused by later work on the same stream
            T = _lib.AVAIL_TILE
            n_tiles = -(-L.nx // T) * -(-L.ny // T)
            seg_d = self._h2d(sg, np.float64)
            tile_cnt = torch.zeros(n_tiles, dtype=torch.int32, device=self.dev)
            g.segs, g.n_segs, g.tile_cnt = seg_d.data_ptr(), len(sg), tile_cnt.data_ptr()
            _lib.check(self.lib.atl_avail_geom_bin(self.device, C.byref(g), row0, 0, _stream_ptr()))
            tile_ptr = torch.zeros(n_tiles + 1, dtype=torch.int64, device=self.dev)
            torch.cumsum(tile_cnt, 0, out=tile_ptr[1:])
            cursor = tile_ptr[:-1].clone()
            tile_list = torch.empty(max(int(tile_ptr[-1]), 1), dtype=torch.int32, device=self.dev)
            g.tile_cursor, g.tile_ptr, g.tile_list = cursor.data_ptr(), tile_ptr.data_ptr(), tile_list.data_ptr()
            _lib.check(self.lib.atl_avail_geom_bin(self.device, C.byref(g), row0, 1, _stream_ptr()))
        _lib.check(self.lib.atl_avail_geometry(self.device, C.byref(g), row0, _stream_ptr()))

    # ---- results
    def shape_mask(self, parts):
        out = transform = None
        for excl, _, j0, transform, shape in self.bands(parts):
            if out is None:
                out = np.empty(shape, dtype=bool)
            out[j0:j0 + excl.shape[0]] = (excl == 0).cpu().numpy()
        return out, transform

    def _average_desc(self, parts, dst, dst_crs):
        """The AtlAvailAverage of one shape's window onto the grid ``dst`` (a ``_lib.Lattice``) in
        ``dst_crs``, its rectangle still unset."""
        b = parts.bounds()
        if b is None:
            raise ValueError("a shape without polygon parts has no availability window")
        transform, (ny, nx) = padded_transform_and_shape(b, self.res)
        _, _, left, _, _, top = _coeffs(transform)
        A = _lib.AvailAverage()
        A.win, A.dst = _lattice(left, self.res, top, -self.res, nx, ny), dst
        A.proj = proj.device_projection(dst_crs, self.crs)  # destination points into the window's CRS
        A.pad = reprojection_pad(transform, self.crs, dst.a, dst_crs)
        return A

    def average(self, parts, dst, dst_crs):
        """float64 NumPy (dst.ny, dst.nx): the eligible share of each cell of ``dst`` (a ``_lib.Lattice``
        in ``dst_crs``), the padded window's mask averaged over each cell's footprint.  One box pass
        over the grid finds the rectangle of cells the window reaches; only its cells are counted,
        band by band, and finalized; every other cell is 0."""
        from .engine import ReprojectOp

        torch = self.torch
        A = self._average_desc(parts, dst, dst_crs)
        rect_d = torch.empty(4, dtype=torch.int32, device=self.dev)
        rect = (C.c_int32 * 4)()
        _lib.check(self.lib.atl_avail_average_rect(self.device, C.byref(A), _dptr(rect_d), rect, _stream_ptr()))
        r0, c0, r1, c1 = (int(v) for v in rect)
        A.row0, A.col0, A.row1, A.col1 = r0, c0, r1, c1
        W = A.win
        A.tile_y, A.tile_x = ReprojectOp._tile(
            ((W.a, 0.0, W.c, 0.0, W.e, W.f), (W.ny, W.nx), self.crs),
            ((dst.a, 0.0, dst.c + c0 * dst.a, 0.0, dst.e, dst.f + r0 * dst.e), (r1 - r0, c1 - c0), proj.epsg(dst_crs)))
        counts = torch.zeros(((r1 - r0) * (c1 - c0), 9), dtype=torch.int64, device=self.dev)
        for excl, _, j0, _, _ in self.bands(parts):  # every band runs, so a shape's errors do not depend on dst
            if len(counts):
                _lib.check(self.lib.atl_avail_average_counts(self.device, C.byref(A), _dptr(excl), j0, excl.shape[0],
                                                             _dptr(counts), _stream_ptr()))
        out = np.zeros((dst.ny, dst.nx))
        if len(counts):
            vals = torch.empty((r1 - r0, c1 - c0), dtype=torch.float64, device=self.dev)
            _lib.check(self.lib.atl_avail_average_finalize(self.device, C.byref(A), _dptr(counts), _dptr(vals),
                                                           _stream_ptr()))
            out[r0:r1, c0:c1] = vals.cpu().numpy()
        return out

    def average_corners(self, parts, dst, dst_crs):
        """(dst.ny + 1, dst.nx + 1, 2) float64: the window pixel coordinates (u, v) of ``dst``'s lattice
        points as the average's kernels compute them (NaN without an image)."""
        A = self._average_desc(parts, dst, dst_crs)
        uv = self.torch.empty((dst.ny + 1, dst.nx + 1, 2), dtype=self.torch.float64, device=self.dev)
        _lib.check(self.lib.atl_avail_average_corners(self.device, C.byref(A), _dptr(uv), _stream_ptr()))
        return uv.cpu().numpy()

    def counts(self, shape_parts, grid, cutout_crs):
        gx0, gdx, gy0, gdy, gnx, gny = grid
        torch = self.torch
        out = torch.zeros((len(shape_parts), gny, gnx), dtype=torch.int64, device=self.dev)
        P = proj.device_projection(self.crs, cutout_crs)
        for k, parts in enumerate(shape_parts):
            if parts.bounds() is None:
                continue
            for excl, L, j0, _, _ in self.bands(parts):
                c = _lib.AvailCount()
                c.win, c.proj, c.win_row0, c.excl = L, P, j0, excl.data_ptr()
                c.gx0, c.gdx, c.gy0, c.gdy, c.gnx, c.gny = float(gx0), float(gdx), float(gy0), float(gdy), gnx, gny
                c.counts = out[k].data_ptr()
                _lib.check(self.lib.atl_avail_count(self.device, C.byref(c), _stream_ptr()))
        return out.cpu().numpy()
