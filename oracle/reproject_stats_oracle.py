"""CPU oracle for the statistics of ``atlite_b200.gis.reproject`` / ``gis.regrid`` (TEST INFRASTRUCTURE
ONLY -- never imported by atlite_b200): sum, rms, min, max, med, q1, q3 and mode (rasterio's
Resampling 13, 14, 9, 8, 10, 11, 12, 6).

A float64 NumPy restatement of DESIGN.md section 1, written cell by cell:

  * a cell's pixels and weights are the average's: across CRSs the two-corner box (the corners
    projected with ``reproject_oracle._to_source``), along each axis the pixels
    ``floor(t0 + EPS) <= k < ceil(t1 - EPS)`` inside the source, each weighted by its overlap
    ``min(k + 1, t1) - max(k, t0)``; within one CRS the rows and columns of ``gis.regrid_axis``
    tables with their weights.  ``w = w_v * w_u``.  A pixel is valid when it is neither NaN nor
    ``src_nodata``; a cell without an image or without a valid pixel gets ``dst_nodata``;
  * sum = sum w v, rms = sqrt(sum w v^2 / sum w) (float64, then rounded once to the dtype);
  * min / max: the smallest / largest valid value, -0.0 below +0.0, bit for bit;
  * med, q1, q3, mode with q = llround(w 2^40) in Python integers, -0.0 counted as +0.0:
    the smallest valid x with 4 C(x) >= k W (k = 2, 1, 3), and the value of the largest sum of q
    (ties to the smaller value); W = 0 gives ``dst_nodata``.

Small cases only.
"""

from __future__ import annotations

import math

import numpy as np

import reproject_oracle as RO

MODE, MAX, MIN, MED, Q1, Q3, SUM, RMS = 6, 8, 9, 10, 11, 12, 13, 14
STATS = (MODE, MAX, MIN, MED, Q1, Q3, SUM, RMS)
SELECT_K = {Q1: 1, MED: 2, Q3: 3}


def axis_pixels(t0, t1, n):
    """(indices, overlaps) of the pixels of [t0, t1] along an axis of n pixels (footprint.cuh)."""
    lo = int(min(max(math.floor(t0 + RO.EPS), 0), n))
    hi = int(min(max(math.ceil(t1 - RO.EPS), 0), n))
    k = np.arange(lo, hi)
    return k, np.minimum(k + 1.0, t1) - np.maximum(k.astype(np.float64), t0)


def corner_boxes(src_t, src_crs, src_shape, dst_t, dst_crs, dst_shape):
    """{(i, j): (rows, wy, cols, wx)} of the two-corner boxes; cells without an image are left out."""
    a, _, c, _, e, f = (float(t) for t in tuple(dst_t)[:6])
    out = {}
    for i in range(dst_shape[0]):
        for j in range(dst_shape[1]):
            u0, v0 = RO._to_source(c + j * a, f + i * e, src_t, src_crs, dst_crs)
            u1, v1 = RO._to_source(c + (j + 1) * a, f + (i + 1) * e, src_t, src_crs, dst_crs)
            if not all(math.isfinite(t) for t in (u0, v0, u1, v1)):
                continue
            rows, wy = axis_pixels(min(v0, v1), max(v0, v1), src_shape[0])
            cols, wx = axis_pixels(min(u0, u1), max(u0, u1), src_shape[1])
            out[i, j] = rows, wy, cols, wx
    return out


def table_boxes(ytab, xtab):
    """{(i, j): (rows, wy, cols, wx)} of ``regrid_axis`` tables (y, x) over the stored source order."""
    (yf, yc, yw), (xf, xc, xw) = ytab, xtab
    return {(i, j): (np.arange(yf[i], yf[i] + yc[i]), np.asarray(yw[i, :yc[i]], dtype=np.float64),
                     np.arange(xf[j], xf[j] + xc[j]), np.asarray(xw[j, :xc[j]], dtype=np.float64))
            for i in range(len(yf)) for j in range(len(xf))}


def _uint(dtype):
    return np.uint32 if np.dtype(dtype) == np.float32 else np.uint64


def order_keys(v):
    """Unsigned keys in the order of the values ``v`` (-0.0 below +0.0)."""
    u = np.ascontiguousarray(v).view(_uint(v.dtype))
    sign = _uint(v.dtype)(1) << _uint(v.dtype)(8 * v.dtype.itemsize - 1)
    return np.where(u & sign, ~u, u | sign)


def weight_q(w):
    """llround(w * 2^40) as Python ints (w >= 0)."""
    return [int(math.floor(x + 0.5)) for x in (np.asarray(w, dtype=np.float64) * 2.0 ** 40).tolist()]


def cell_stat(win, w, code, src_nodata=None):
    """The statistic ``code`` of one cell: ``win`` its pixel values (any shape, float32 / float64),
    ``w`` their float64 weights.  None when the cell gets dst_nodata."""
    win, w = np.asarray(win).ravel(), np.asarray(w, dtype=np.float64).ravel()
    ok = ~RO._skip(win, src_nodata)
    vals, w = win[ok], w[ok]
    if not len(vals):
        return None
    if code in (SUM, RMS):
        v = vals.astype(np.float64)
        s = float(np.sum(w * (v * v if code == RMS else v)))
        return s if code == SUM else math.sqrt(s / float(np.sum(w)))
    if code in (MIN, MAX):
        k = order_keys(vals)
        return vals[int(np.argmin(k) if code == MIN else np.argmax(k))]
    zero = vals == 0  # -0.0 counts as +0.0
    vals = np.where(zero, np.zeros_like(vals), vals)
    q = weight_q(w)
    keys = order_keys(vals).tolist()
    tot = {}
    val_of = {}
    for key, qq, x in zip(keys, q, vals):
        tot[key] = tot.get(key, 0) + qq
        val_of[key] = x
    W = sum(tot.values())
    if W == 0:
        return None
    order = sorted(tot)
    if code == MODE:
        best = max(tot.values())
        return val_of[next(k for k in order if tot[k] == best)]
    need, c = SELECT_K[code] * W, 0
    for key in order:
        c += tot[key]
        if 4 * c >= need:
            return val_of[key]
    raise AssertionError("unreachable: 4 C reaches 4 W")


def resample(values, boxes, dst_shape, code, src_nodata=None, dst_nodata=None):
    """``values`` (..., ny, nx) -> (..., *dst_shape): float64 for sum / rms, the values' dtype
    otherwise.  ``boxes`` from ``corner_boxes`` or ``table_boxes``."""
    v = np.asarray(values)
    if dst_nodata is None:
        dst_nodata = src_nodata if src_nodata is not None else np.nan
    dtype = np.float64 if code in (SUM, RMS) else v.dtype
    lead = v.shape[:-2]
    out = np.full(lead + tuple(dst_shape), dst_nodata, dtype=dtype)
    for (i, j), (rows, wy, cols, wx) in boxes.items():
        if not len(rows) or not len(cols):
            continue
        w = wy[:, None] * wx[None, :]
        for idx in np.ndindex(*lead):
            res = cell_stat(v[idx][np.ix_(rows, cols)], w, code, src_nodata)
            if res is not None:
                out[idx + (i, j)] = res
    return out


def reproject(values, src_t, src_crs, dst_t, dst_crs, dst_shape, code, src_nodata=None, dst_nodata=None):
    """The statistic of ``gis.reproject`` across CRSs (or on the identity pair)."""
    boxes = corner_boxes(src_t, src_crs, np.shape(values)[-2:], dst_t, dst_crs, dst_shape)
    return resample(values, boxes, dst_shape, code, src_nodata, dst_nodata)
