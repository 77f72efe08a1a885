"""CPU oracle for ``atlite_b200.gis.reproject`` (TEST INFRASTRUCTURE ONLY -- never imported by atlite_b200).

float64 NumPy restatement of the "reproject semantics" of DESIGN.md section 1, written cell by cell:

  * source pixel coordinates of a point are ``u = (x - c) / a``, ``v = (y - f) / e`` (the inverse of
    the source's axis-aligned affine transform, either sign of a and e);
  * average: destination cell (i, j) projects its own two corners ``T_dst (j, i)`` and
    ``T_dst (j + 1, i + 1)`` from the destination CRS into the source CRS with ``proj.transform`` and
    takes them to (u, v); the footprint is the box they span.  Every source pixel inside the source
    whose overlap with the box exceeds ``EPS`` along both axes takes the weight
    ``overlap_u * overlap_v``; NaN and ``src_nodata`` are skipped; the weighted mean is summed along
    x, then along y; a cell with no valid pixel, or a corner without an image, gets ``dst_nodata``;
  * nearest: the centre ``T_dst (j + 1/2, i + 1/2)`` is projected and floored; inside the source the
    cell takes that pixel (NaN and nodata become ``dst_nodata``), outside it gets ``dst_nodata``.

It shares no code with atlite_b200 beyond ``proj``'s formulas, which define the CRSs.  Small cases only.
"""

from __future__ import annotations

import math

import numpy as np

from atlite_b200 import proj

EPS = 1e-10


def _to_source(x, y, src_t, src_crs, dst_crs):
    a, _, c, _, e, f = src_t
    px, py = proj.transform(np.float64(x), np.float64(y), dst_crs, src_crs)
    return (float(px) - c) / a, (float(py) - f) / e


def _skip(v, src_nodata):
    return np.isnan(v) | ((v == src_nodata) if src_nodata is not None else False)


def reproject(values, src_t, src_crs, dst_t, dst_crs, dst_shape, resampling=5, src_nodata=None, dst_nodata=None):
    """``values`` (..., ny, nx) on the source grid -> (..., *dst_shape) float64.  Transforms are
    6-tuples (a, 0, c, 0, e, f)."""
    v = np.asarray(values, dtype=np.float64)
    ny, nx = v.shape[-2:]
    if dst_nodata is None:
        dst_nodata = src_nodata if src_nodata is not None else np.nan
    a, _, c, _, e, f = (float(t) for t in tuple(dst_t)[:6])
    out = np.full(v.shape[:-2] + tuple(dst_shape), float(dst_nodata))
    for i in range(dst_shape[0]):
        for j in range(dst_shape[1]):
            if resampling == 0:
                u, w = _to_source(c + (j + 0.5) * a, f + (i + 0.5) * e, src_t, src_crs, dst_crs)
                if not (math.isfinite(u) and math.isfinite(w)):
                    continue
                col, row = math.floor(u), math.floor(w)
                if 0 <= col < nx and 0 <= row < ny:
                    px = v[..., row, col]
                    out[..., i, j] = np.where(_skip(px, src_nodata), dst_nodata, px)
                continue
            u0, v0 = _to_source(c + j * a, f + i * e, src_t, src_crs, dst_crs)
            u1, v1 = _to_source(c + (j + 1) * a, f + (i + 1) * e, src_t, src_crs, dst_crs)
            if not all(math.isfinite(t) for t in (u0, v0, u1, v1)):
                continue
            u0, u1 = sorted((u0, u1))
            v0, v1 = sorted((v0, v1))
            cs = np.arange(max(0, math.floor(u0) - 1), min(nx, math.ceil(u1) + 1))
            rs = np.arange(max(0, math.floor(v0) - 1), min(ny, math.ceil(v1) + 1))
            cs = cs[(np.minimum(cs + 1.0, u1) - np.maximum(cs.astype(np.float64), u0) > EPS)]
            rs = rs[(np.minimum(rs + 1.0, v1) - np.maximum(rs.astype(np.float64), v0) > EPS)]
            if not len(cs) or not len(rs):
                continue
            ox = np.minimum(cs + 1.0, u1) - np.maximum(cs.astype(np.float64), u0)
            oy = np.minimum(rs + 1.0, v1) - np.maximum(rs.astype(np.float64), v0)
            win = v[..., rs[:, None], cs[None, :]]
            ok = ~_skip(win, src_nodata)
            den = (oy[:, None] * ox[None, :] * ok).sum(axis=-1).sum(axis=-1)
            num = (oy[:, None] * ox[None, :] * np.where(ok, win, 0.0)).sum(axis=-1).sum(axis=-1)
            with np.errstate(invalid="ignore", divide="ignore"):
                out[..., i, j] = np.where(den > 0, num / np.where(den > 0, den, 1.0), dst_nodata)
    return out


def centre_edge_distance(src_t, src_crs, dst_t, dst_crs, dst_shape):
    """(ny, nx) distance in source pixels from each destination centre's (u, v) to the nearest pixel
    edge (NaN where the centre has no image): nearest resampling is ambiguous where it is ~0."""
    a, _, c, _, e, f = (float(t) for t in tuple(dst_t)[:6])
    d = np.full(tuple(dst_shape), np.nan)
    for i in range(dst_shape[0]):
        for j in range(dst_shape[1]):
            u, w = _to_source(c + (j + 0.5) * a, f + (i + 0.5) * e, src_t, src_crs, dst_crs)
            if math.isfinite(u) and math.isfinite(w):
                d[i, j] = min(abs(u - round(u)), abs(w - round(w)))
    return d
