"""GEBCO terrain height for a cutout (datasets/gebco.py of the reference).

``get_data`` reads the window of a GEBCO grid (NetCDF, 15 arc-second ``elevation``, int16) that the
cutout covers and averages it onto the cutout's cells: ``ingest.open_grid`` slices the window out of
the file without loading the rest, and the average runs on the GPU (``engine.RegridOp.window``,
csrc/regrid.cu), which streams host windows in bands of rows.  ``raster`` cuts a window as a
``gis.Raster`` for ``ExclusionContainer.add_raster`` (depth exclusion without rasterio).
Semantics and deviations: DESIGN.md section 1.
"""

from __future__ import annotations

import logging
import math

import numpy as np

logger = logging.getLogger(__name__)

# CRS and features (datasets/gebco.py:19-20)
crs = 4326
features = {"height": ["height"]}


def grid_transform(lon, lat):
    """The north-up affine transform ``(a, 0, c, 0, e, f)`` GDAL's netCDF driver builds from the
    grid's ``lon`` / ``lat`` centres: pixel size ``(last - first) / (n - 1)``, origin half a pixel
    out from the first column's centre and the northernmost row's centre."""
    from .gis import regular_axis

    lon0, a = regular_axis(lon, "lon")
    lat = np.asarray(lat, dtype=np.float64)
    _, dlat = regular_axis(lat[::-1] if len(lat) > 1 and lat[-1] < lat[0] else lat, "lat")
    e = -dlat
    return (a, 0.0, lon0 - a / 2, 0.0, e, float(max(lat[0], lat[-1])) - e / 2)


def window(transform, left, bottom, right, top):
    """(col_off, row_off, width, height) in pixels of the bounds in the grid of ``transform``, as
    rasterio's ``windows.from_bounds`` computes them: the four corners through the inverse affine
    transform, then their least and greatest column and row."""
    a, _, c, _, e, f = transform
    idet = 1.0 / (a * e)
    ra, re = e * idet, a * idet
    cols = [x * ra + -c * ra for x in (left, right, right, left)]
    rows = [y * re + -f * re for y in (top, top, bottom, bottom)]
    col_off, row_off = min(cols), min(rows)
    return col_off, row_off, max(max(cols) - col_off, 0.0), max(max(rows) - row_off, 0.0)


def _cutout_window(xs, ys, transform, shape):
    """The reference's window for cutout centres ``xs`` / ``ys`` (datasets/gebco.py:24-31), checked
    to lie inside a grid of ``shape`` (rows, columns)."""
    from .gis import REGRID_EPS

    xs, ys = np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64)
    for name, c in (("x", xs), ("y", ys)):
        if c.ndim != 1 or len(c) < 2:
            raise ValueError(f"the cutout needs at least 2 cells along {name!r}, not {c.size}")
        if not c[-1] > c[0]:
            raise ValueError(f"the cutout's {name!r} coordinates must ascend")
    (x, X), (y, Y) = xs[[0, -1]], ys[[0, -1]]
    dx, dy = (X - x) / (len(xs) - 1), (Y - y) / (len(ys) - 1)
    win = window(transform, x - dx / 2, y - dy / 2, X + dx / 2, Y + dy / 2)
    col_off, row_off, width, height = win
    if (col_off < -REGRID_EPS or row_off < -REGRID_EPS or col_off + width > shape[1] + REGRID_EPS
            or row_off + height > shape[0] + REGRID_EPS):
        raise ValueError(f"the cutout's extent ({x - dx / 2}, {y - dy / 2}, {X + dx / 2}, {Y + dy / 2}) is not inside "
                         f"the GEBCO grid: window (col_off, row_off, width, height) {win} of {shape[1]} x {shape[0]}")
    return win


def _tables(win, nx, ny, shape, lat_ascending):
    """(rows, cols, ytab, xtab): the file rows and columns of the window the cells read, and the
    regrid tables of the cells relative to them, destination rows in ascending y.  Cell j spans
    pixels ``[col_off + j * width / nx, col_off + (j + 1) * width / nx]`` (north-up rows alike),
    with ``regrid``'s fractional weights and 1e-10 sliver rule and no padding."""
    from .gis import _flip_axis_table, regrid_axis

    col_off, row_off, width, height = win
    sx, sy = width / nx, height / ny
    xtab = regrid_axis(0.5, 1.0, shape[1], col_off + sx / 2, sx, nx, 0)
    ytab = regrid_axis(0.5, 1.0, shape[0], row_off + sy / 2, sy, ny, 0)  # north-up rows
    if lat_ascending:  # north-up row R is file row n - 1 - R
        ytab = _flip_axis_table(ytab, shape[0])
    ytab = tuple(np.ascontiguousarray(t[::-1]) for t in ytab)  # north-up cells -> ascending y

    def span(tab):
        first, count, w = tab
        lo, hi = int(first[count > 0].min()), int((first + count)[count > 0].max())
        return (lo, hi), (np.where(count > 0, first - lo, 0).astype(np.int32), count, w)

    rows, ytab = span(ytab)
    cols, xtab = span(xtab)
    return rows, cols, ytab, xtab


def get_data_gebco_height(xs, ys, gebco_path):
    """``height(y, x)``: the GEBCO grid averaged onto the cells with centres ``xs`` / ``ys``
    (ascending, at least 2 each; datasets/gebco.py:23-44), as this package's ``DataArray`` whose attrs
    are the variable's attributes.  The dtype is the file's: int16 means are rounded half away from
    zero.  Pixels equal to the fill value are skipped; a cell made only of them gets the fill value."""
    from . import ingest
    from .engine import RegridOp, current_device
    from .labelled import DataArray

    xs, ys = np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64)
    lon, lat, var = ingest.open_grid(gebco_path)
    win = _cutout_window(xs, ys, grid_transform(lon, lat), var.shape)
    (r0, r1), (c0, c1), ytab, xtab = _tables(win, len(xs), len(ys), var.shape, lat[-1] > lat[0])
    op = RegridOp((r1 - r0, c1 - c0), ytab, xtab, device=current_device())
    height = op.window(var.window(r0, r1, c0, c1), fill=var.fill)
    return DataArray(height, {"y": ys, "x": xs}, ("y", "x"), "height", dict(var.attrs))


def get_data(cutout, feature, tmpdir, monthly_requests=False, concurrent_requests=False, **creation_parameters):
    """GEBCO ``height`` for ``cutout`` (datasets/gebco.py:47-89): a host-resident Dataset with
    ``height(y, x)`` and the cutout's coordinates, ready for ``Cutout.merge``; an xarray Dataset,
    with the variable's attributes on ``height``, when the cutout's data is one.
    ``creation_parameters`` must hold ``gebco_path``; ``tmpdir``, ``monthly_requests`` and
    ``concurrent_requests`` are accepted and unused.  ``feature`` must be ``"height"``, GEBCO's
    only feature."""
    from .labelled import HAVE_XARRAY, Dataset, xr

    if feature != "height":
        raise ValueError(f"GEBCO provides the feature 'height' only, not {feature!r}")
    if "gebco_path" not in creation_parameters:
        logger.error('Argument "gebco_path" not defined')
        raise KeyError("gebco_path: GEBCO's get_data needs the creation parameter 'gebco_path'")
    coords = cutout.coords
    h = get_data_gebco_height(coords["x"], coords["y"], creation_parameters["gebco_path"])
    if HAVE_XARRAY and isinstance(cutout.data, xr.Dataset):  # pragma: no cover - xarray is optional
        ds = xr.Dataset({"height": (("y", "x"), h.values, h.attrs)}, attrs={"module": "gebco"})
        return ds.assign_coords(cutout.data.coords)
    return Dataset({"height": (("y", "x"), h.values)}, coords=dict(coords), attrs={"module": "gebco"})


def raster(gebco_path, bounds=None):
    """The GEBCO window covering ``bounds`` = (left, bottom, right, top) in lon / lat (None: the
    whole grid) as a north-up ``gis.Raster(int16 values, transform, 4326)``, read without loading
    the rest of the file: every pixel the bounds overlap (by more than 1e-10 pixel), clipped to the
    grid.  For example ``ExclusionContainer.add_raster(gebco.raster(path, bounds), codes=lambda h:
    h < -50, crs=4326)`` excludes water deeper than 50 m."""
    from . import ingest
    from .gis import REGRID_EPS, Raster

    lon, lat, var = ingest.open_grid(gebco_path)
    t = grid_transform(lon, lat)
    nrows, ncols = var.shape
    if bounds is None:
        (c0, c1), (n0, n1) = (0, ncols), (0, nrows)
    else:
        col_off, row_off, width, height = window(t, *(float(b) for b in bounds))
        c0, c1 = max(0, math.floor(col_off + REGRID_EPS)), min(ncols, math.ceil(col_off + width - REGRID_EPS))
        n0, n1 = max(0, math.floor(row_off + REGRID_EPS)), min(nrows, math.ceil(row_off + height - REGRID_EPS))
        if c1 <= c0 or n1 <= n0:
            raise ValueError(f"bounds {tuple(bounds)} do not overlap the GEBCO grid")
    if lat[-1] > lat[0]:  # north-up rows [n0, n1) are file rows [nrows - n1, nrows - n0), reversed
        arr = np.ascontiguousarray(var[nrows - n1:nrows - n0, c0:c1][::-1])
    else:
        arr = var[n0:n1, c0:c1]
    a, _, c, _, e, f = t
    return Raster(arr, (a, 0.0, c + c0 * a, 0.0, e, f + n0 * e), crs)
