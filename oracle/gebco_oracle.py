"""CPU oracle for ``atlite_b200.gebco`` (TEST INFRASTRUCTURE ONLY -- never imported by atlite_b200).

float64 NumPy restatement of the GEBCO semantics in DESIGN.md section 1, written cell by cell:

  * the grid's north-up transform from its centres: pixel size ``(last - first) / (n - 1)``, origin
    half a pixel out from the first column and the northernmost row;
  * the window of the cutout's extent ``(x - dx/2, y - dy/2, X + dx/2, Y + dy/2)`` as rasterio's
    ``windows.from_bounds`` computes it (the corners through the inverse affine transform);
  * cell j along an axis spans pixels ``[off + j * size / n, off + (j + 1) * size / n]`` of the
    window's north-up rows / columns, no padding; the output is flipped to ascending y;
  * every cell gathers its own rectangle of pixels with overlap-length weights (an overlap of
    1e-10 pixel or less does not count) and takes the weighted mean of the pixels that are neither
    NaN nor the fill value; the fill value (else NaN) without one.

It returns the unrounded float64 means; the int16 result is their rounding half away from zero.
"""

from __future__ import annotations

import math

import numpy as np

EPS = 1e-10


def transform(lon, lat):
    lon, lat = np.asarray(lon, dtype=np.float64), np.asarray(lat, dtype=np.float64)
    a = (lon[-1] - lon[0]) / (len(lon) - 1)
    dlat = abs(lat[-1] - lat[0]) / (len(lat) - 1)
    return a, 0.0, lon[0] - a / 2, 0.0, -dlat, max(lat[0], lat[-1]) + dlat / 2


def from_bounds(t, left, bottom, right, top):
    """rasterio.windows.from_bounds: (col_off, row_off, width, height)."""
    a, b, c, d, e, f = t
    idet = 1.0 / (a * e - b * d)
    ra, rb, rd, re = e * idet, -b * idet, -d * idet, a * idet
    rc, rf = -c * ra - f * rb, -c * rd - f * re
    xs, ys = np.array([left, right, right, left]), np.array([top, top, bottom, bottom])
    cols, rows = xs * ra + ys * rb + rc, xs * rd + ys * re + rf
    return cols.min(), rows.min(), max(cols.max() - cols.min(), 0.0), max(rows.max() - rows.min(), 0.0)


def cutout_window(lon, lat, xs, ys):
    x, X = np.asarray(xs, dtype=np.float64)[[0, -1]]
    y, Y = np.asarray(ys, dtype=np.float64)[[0, -1]]
    dx, dy = (X - x) / (len(xs) - 1), (Y - y) / (len(ys) - 1)
    return from_bounds(transform(lon, lat), x - dx / 2, y - dy / 2, X + dx / 2, Y + dy / 2)


def _overlaps(u0, u1, n):
    k = np.arange(max(0, math.floor(u0) - 1), min(n, math.ceil(u1) + 1))
    w = np.minimum(k + 1.0, u1) - np.maximum(k.astype(np.float64), u0)
    keep = w > EPS
    return k[keep], w[keep]


def height(elevation, lon, lat, xs, ys, fill=None):
    """(len(ys), len(xs)) float64 means of ``elevation`` (lat, lon as stored) on the cutout cells."""
    v = np.asarray(elevation, dtype=np.float64)
    lat = np.asarray(lat, dtype=np.float64)
    if lat[-1] > lat[0]:
        v = v[::-1]  # north-up
    nrows, ncols = v.shape
    col_off, row_off, width, hgt = cutout_window(lon, lat, xs, ys)
    nx, ny = len(xs), len(ys)
    sx, sy = width / nx, hgt / ny
    out = np.empty((ny, nx))
    for i in range(ny):
        rows, wy = _overlaps(row_off + i * sy, row_off + (i + 1) * sy, nrows)
        for j in range(nx):
            cols, wx = _overlaps(col_off + j * sx, col_off + (j + 1) * sx, ncols)
            win = v[rows[:, None], cols[None, :]]
            ok = ~np.isnan(win)
            if fill is not None:
                ok &= win != fill
            area = wy[:, None] * wx[None, :] * ok
            den = area.sum()
            out[ny - 1 - i, j] = (area * np.where(ok, win, 0.0)).sum() / den if den > 0 else (
                np.nan if fill is None else fill)
    return out


def round_half_away(m):
    return np.sign(m) * np.floor(np.abs(m) + 0.5)
