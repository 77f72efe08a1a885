"""CPU oracle for ``atlite_b200.regrid`` (TEST INFRASTRUCTURE ONLY -- never imported by atlite_b200).

float64 NumPy restatement of the semantics in DESIGN.md section 1 (the reference's gis.py:765-871
with rasterio's average and nearest resampling in one CRS), written cell by cell:

  * the source is flipped to ascending axes; its pixel k along an axis covers
    ``[first - step / 2 + k * step, first - step / 2 + (k + 1) * step]`` with
    ``step = (last - first) / (n - 1)``, the destination's cells are built the same way from
    ``dimx`` / ``dimy`` in their given order;
  * the source is padded by ``pad = int(|dst dx| // min(src dx, src dy) * 1.1)`` pixels on every
    side, each padded pixel repeating the nearest border pixel;
  * average: for every destination cell, the 2-D overlap of the cell with every padded source
    pixel, in source pixels (an overlap shorter than ``EPS`` along either axis does not count),
    and the overlap-weighted mean of the non-NaN values; NaN without one;
  * nearest: the padded pixel containing the cell centre (a centre on a border takes the pixel on
    the increasing-coordinate side); NaN outside the padded source.

It does not use atlite_b200's separable per-axis tables: every cell gathers its own rectangle of
padded pixels.  Small cases only.
"""

from __future__ import annotations

import math

import numpy as np

EPS = 1e-10


def _axis(c):
    c = np.asarray(c, dtype=np.float64)
    return float(c[0]), float(c[-1] - c[0]) / float(len(c) - 1)


def regrid(values, xs, ys, dimx, dimy, resampling=5):
    """``values`` (..., len(ys), len(xs)) on the source centres ``xs`` / ``ys`` (either order) ->
    (..., len(dimy), len(dimx)) float64 on the destination centres, ``resampling`` 5 (average) or 0
    (nearest)."""
    v = np.asarray(values, dtype=np.float64)
    xs, ys = np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64)
    if xs[-1] < xs[0]:
        v, xs = v[..., ::-1], xs[::-1]
    if ys[-1] < ys[0]:
        v, ys = v[..., ::-1, :], ys[::-1]
    nys, nxs = len(ys), len(xs)
    sx0, sdx = _axis(xs)
    sy0, sdy = _axis(ys)
    dx0, ddx = _axis(dimx)
    dy0, ddy = _axis(dimy)
    pad = int(abs(ddx) // min(sdx, sdy) * 1.1)
    sox, soy = sx0 - sdx / 2, sy0 - sdy / 2
    dox, doy = dx0 - ddx / 2, dy0 - ddy / 2
    out = np.full(v.shape[:-2] + (len(dimy), len(dimx)), np.nan)

    for i in range(len(dimy)):
        for j in range(len(dimx)):
            if resampling == 0:
                c = math.floor((dox + (j + 0.5) * ddx - sox) / sdx)
                r = math.floor((doy + (i + 0.5) * ddy - soy) / sdy)
                if -pad <= c < nxs + pad and -pad <= r < nys + pad:
                    out[..., i, j] = v[..., min(max(r, 0), nys - 1), min(max(c, 0), nxs - 1)]
                continue
            x0, x1 = sorted((dox + j * ddx, dox + (j + 1) * ddx))
            y0, y1 = sorted((doy + i * ddy, doy + (i + 1) * ddy))
            ux0, ux1 = (x0 - sox) / sdx, (x1 - sox) / sdx
            uy0, uy1 = (y0 - soy) / sdy, (y1 - soy) / sdy
            cs = np.arange(max(-pad, math.floor(ux0) - 1), min(nxs + pad, math.ceil(ux1) + 1))
            rs = np.arange(max(-pad, math.floor(uy0) - 1), min(nys + pad, math.ceil(uy1) + 1))
            cs = cs[(cs + 1 - ux0 > EPS) & (ux1 - cs > EPS)]
            rs = rs[(rs + 1 - uy0 > EPS) & (uy1 - rs > EPS)]
            if not len(cs) or not len(rs):
                continue
            ox = np.minimum(cs + 1.0, ux1) - np.maximum(cs.astype(np.float64), ux0)
            oy = np.minimum(rs + 1.0, uy1) - np.maximum(rs.astype(np.float64), uy0)
            area = oy[:, None] * ox[None, :]
            win = v[..., np.clip(rs, 0, nys - 1)[:, None], np.clip(cs, 0, nxs - 1)[None, :]]
            ok = ~np.isnan(win)
            den = (area * ok).sum(axis=-1).sum(axis=-1)  # along x, then y: the same order for any leading dims
            num = (area * np.where(ok, win, 0.0)).sum(axis=-1).sum(axis=-1)
            with np.errstate(invalid="ignore", divide="ignore"):
                out[..., i, j] = np.where(den > 0, num / np.where(den > 0, den, 1.0), np.nan)
    return out
