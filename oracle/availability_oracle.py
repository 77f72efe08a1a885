"""NumPy oracle of the land-eligibility specification (atlite_b200/availability.py), float64.

Pixel (i, j) of a lattice (c, a, f, e) has its centre at x = c + (i + 0.5) a, y = f + (j + 0.5) e.
Polygon masks are decided exactly: a centre is left of an edge by the sign of orient2d, from a float
filter with Shewchuk's bound and exact rational arithmetic when the filter cannot decide, so the
masks must equal the GPU's bit for bit.  Where a decision rests on a projected pixel centre or a
float distance, the oracle also returns the pixels whose decision lies within 1e-9 (relative) of a
tie; those are the only ones a comparison may excuse.

Polygon vertices and pixel centres are projected with ``atlite_b200.proj`` on the host (vertices are
projected there by the package too, so windows and masks are bit-identical); ``laea_forward`` /
``laea_inverse`` below restate EPSG method 9820 independently to check that module.
"""

from __future__ import annotations

from fractions import Fraction

import numpy as np

from atlite_b200 import proj

_EPS = np.finfo(np.float64).eps / 2
_ERR = (3.0 + 16.0 * _EPS) * _EPS
TIE = 1e-9

# ---------------------------------------------------------------- EPSG:3035, restated (GN 7-2, 9820)
_A, _F = 6378137.0, 1 / 298.257222101


def _q(phi, e):
    s = np.sin(phi)
    return (1 - e * e) * (s / (1 - e * e * s * s) - 1 / (2 * e) * np.log((1 - e * s) / (1 + e * s)))


def laea_forward(lon, lat):
    e = np.sqrt(2 * _F - _F * _F)
    phi0, lam0 = np.radians(52.0), np.radians(10.0)
    qp, q0, q = _q(np.pi / 2, e), _q(phi0, e), _q(np.radians(lat), e)
    Rq = _A * np.sqrt(qp / 2)
    b0, b = np.arcsin(q0 / qp), np.arcsin(q / qp)
    D = _A * np.cos(phi0) / np.sqrt(1 - e * e * np.sin(phi0) ** 2) / (Rq * np.cos(b0))
    dl = np.radians(lon) - lam0
    B = Rq * np.sqrt(2 / (1 + np.sin(b0) * np.sin(b) + np.cos(b0) * np.cos(b) * np.cos(dl)))
    return (4321000.0 + B * D * np.cos(b) * np.sin(dl),
            3210000.0 + B / D * (np.cos(b0) * np.sin(b) - np.sin(b0) * np.cos(b) * np.cos(dl)))


def laea_inverse(x, y):
    """Inverse by fixed-point iteration on q(phi) (no series)."""
    e = np.sqrt(2 * _F - _F * _F)
    phi0, lam0 = np.radians(52.0), np.radians(10.0)
    qp, q0 = _q(np.pi / 2, e), _q(phi0, e)
    Rq = _A * np.sqrt(qp / 2)
    b0 = np.arcsin(q0 / qp)
    D = _A * np.cos(phi0) / np.sqrt(1 - e * e * np.sin(phi0) ** 2) / (Rq * np.cos(b0))
    X, Y = np.asarray(x, float) - 4321000.0, np.asarray(y, float) - 3210000.0
    rho = np.hypot(X / D, D * Y)
    C = 2 * np.arcsin(rho / (2 * Rq))
    bp = np.arcsin(np.cos(C) * np.sin(b0) + D * Y * np.sin(C) * np.cos(b0) / rho)
    lam = lam0 + np.arctan2(X * np.sin(C), D * rho * np.cos(b0) * np.cos(C) - D * D * Y * np.sin(b0) * np.sin(C))
    q = qp * np.sin(bp)
    phi = np.arcsin(q / 2)
    for _ in range(30):
        s = np.sin(phi)
        phi = phi + (1 - e * e * s * s) ** 2 / (2 * np.cos(phi)) * (
            q / (1 - e * e) - s / (1 - e * e * s * s) + 1 / (2 * e) * np.log((1 - e * s) / (1 + e * s)))
    return np.degrees(lam), np.degrees(phi)


# ---------------------------------------------------------------- lattice and masks
def window(bounds, res):
    """(left, top, nx, ny) of the padded window (gis.py:186-194)."""
    left, bottom = ((float(b) // res) * res for b in bounds[:2])
    right, top = ((float(b) // res + 1) * res for b in bounds[2:])
    return left, top, int((right - left) / res), int((top - bottom) / res)


def centres(c, a, n):
    return c + (np.arange(n, dtype=np.float64) + 0.5) * a


def _orient_sign(ax, ay, bx, by, px, py):
    left = (ax - px) * (by - py)
    right = (ay - py) * (bx - px)
    det = left - right
    s = np.sign(det)
    unsure = np.abs(det) <= _ERR * (np.abs(left) + np.abs(right))
    for k in np.flatnonzero(np.atleast_1d(unsure)):
        a = [Fraction(float(np.atleast_1d(v)[k] if np.ndim(v) else v)) for v in (ax, ay, bx, by, px, py)]
        d = (a[0] - a[4]) * (a[3] - a[5]) - (a[1] - a[5]) * (a[2] - a[4])
        s[k] = (d > 0) - (d < 0)
    return s


def ring_edges(rings, orient=False):
    """rings: [(ring (N, 2), is_hole)] -> (edges (n, 4), weights)."""
    e, w = [], []
    for r, hole in rings:
        nxt = np.roll(r, -1, axis=0)
        e.append(np.c_[r, nxt])
        s = 1
        if orient:
            area = np.dot(r[:, 0] - r[0, 0], nxt[:, 1] - r[0, 1]) - np.dot(nxt[:, 0] - r[0, 0], r[:, 1] - r[0, 1])
            s = 1 if (area > 0) != hole else -1
        w.append(np.full(len(r), s))
    return (np.concatenate(e), np.concatenate(w)) if e else (np.zeros((0, 4)), np.zeros(0))


def polygon_mask(edges, w, c, a, f, e, nx, ny, nonzero=False):
    """bool (ny, nx): even-odd (or nonzero winding with oriented weights) over the edges; an edge
    counts for the centres of the rows it crosses ((y1 > cy) != (y2 > cy)) strictly left of it."""
    cx, cy = centres(c, a, nx), centres(f, e, ny)
    acc = np.zeros((ny, nx + 1), dtype=np.int64)
    for (x1, y1, x2, y2), wt in zip(edges, w):
        rows = np.flatnonzero((y1 > cy) != (y2 > cy))
        if not len(rows):
            continue
        up = y2 > y1
        ax, ay, bx, by = (x1, y1, x2, y2) if up else (x2, y2, x1, y1)
        yy = cy[rows]
        xi = ax + (yy - ay) * ((bx - ax) / (by - ay))
        i = np.clip(np.ceil((xi - c) / a - 0.5), 0, nx).astype(np.int64)
        for _ in range(nx + 1):  # exact adjustment: i = number of centres strictly left
            dn = (i > 0) & (_orient_sign(ax, ay, bx, by, cx[np.maximum(i - 1, 0)], yy) <= 0)
            upd = (i < nx) & (_orient_sign(ax, ay, bx, by, cx[np.minimum(i, nx - 1)], yy) > 0)
            if not (dn.any() or upd.any()):
                break
            i = i - dn + upd
        np.add.at(acc, (rows, i), wt if up else -wt)
    # pixel i: sum over edges with i* > i
    s = np.cumsum(acc[:, ::-1], axis=1)[:, ::-1][:, 1:]
    return (s != 0) if nonzero else (s % 2 == 1)


def dilate(mask, k):
    """k dilations with the 4-connected cross, border 0 (pure NumPy)."""
    m = np.asarray(mask, dtype=bool).copy()
    for _ in range(k):
        n = m.copy()
        n[1:] |= m[:-1]
        n[:-1] |= m[1:]
        n[:, 1:] |= m[:, :-1]
        n[:, :-1] |= m[:, 1:]
        m = n
    return m


def rule(codes, values):
    if callable(codes):
        return np.asarray(codes(values)).astype(bool)
    if codes is not None and np.size(codes) > 0 and (np.ndim(codes) > 0 or bool(codes)):
        return np.isin(values, codes)
    return values.astype(bool)


def _project_rings(rings, src, dst):
    return [(np.stack(proj.transform(r[:, 0], r[:, 1], src, dst), axis=1), h) for r, h in rings]


def raster_exclusion(rings, crs, L, raster, codes=None, buffer=0, invert=False, nodata=255, allow_no_overlap=False,
                     res=None):
    """(excluded, tie) on the window L = (left, top, nx, ny, res) for one raster dict
    {array, transform (a, 0, c, 0, e, f), epsg}; rings in the container CRS ``crs``."""
    left, top, nx, ny, res = L
    arr = np.asarray(raster["array"])
    a, _, c, _, e, f = raster["transform"]
    rny, rnx = arr.shape
    rr = rings if raster["epsg"] == crs else _project_rings(rings, crs, raster["epsg"])
    v = np.concatenate([r for r, _ in rr])
    bx0, by0, bx1, by1 = v[:, 0].min(), v[:, 1].min(), v[:, 0].max(), v[:, 1].max()
    rl, rb, rrt, rt = c, f + rny * e, c + rnx * a, f
    overlap = bx0 < rrt and bx1 > rl and by0 < rt and by1 > rb
    if not overlap and not allow_no_overlap:
        raise ValueError("Input shapes do not overlap raster.")
    keep = np.zeros((rny, rnx), dtype=bool)
    if overlap:
        i0, i1 = max(int(np.floor((bx0 - c) / a)), 0), min(int(np.floor((bx1 - c) / a)) + 1, rnx)
        j0, j1 = max(int(np.floor((by1 - f) / e)), 0), min(int(np.floor((by0 - f) / e)) + 1, rny)
        if i1 > i0 and j1 > j0:
            ed, w = ring_edges(rr)
            keep[j0:j1, i0:i1] = polygon_mask(ed, w, c + i0 * a, a, f + j0 * e, e, i1 - i0, j1 - j0)
    cx, cy = np.meshgrid(centres(left, res, nx), centres(top, -res, ny))
    px, py = proj.transform(cx, cy, crs, raster["epsg"])
    u, vv = (px - c) / a, (py - f) / e
    tie = np.zeros(u.shape, bool) if raster["epsg"] == crs else (
        (np.abs(u - np.round(u)) <= TIE * np.maximum(1, np.abs(u))) | (np.abs(vv - np.round(vv)) <= TIE * np.maximum(1, np.abs(vv))))
    col, row = np.floor(u), np.floor(vv)
    inside = (col >= 0) & (col < rnx) & (row >= 0) & (row < rny)
    ci, ri = np.where(inside, col, 0).astype(np.int64), np.where(inside, row, 0).astype(np.int64)
    val = arr[ri, ci]
    ok = inside & keep[ri, ci]
    ex = np.where(ok, rule(codes, val), rule(codes, np.asarray([nodata]).astype(arr.dtype))[0])
    if invert:
        ex = ~ex
    if buffer:
        kk = int(buffer / res) + 1
        ex = dilate(ex, kk)
        tie = dilate(tie, kk)
    return ex, tie


def _seg_dist(px, py, s):
    x1, y1, x2, y2 = s
    dx, dy = x2 - x1, y2 - y1
    l2 = dx * dx + dy * dy
    t = np.clip(((px - x1) * dx + (py - y1) * dy) / l2, 0, 1) if l2 > 0 else np.zeros_like(px)
    return np.hypot(px - (x1 + t * dx), py - (y1 + t * dy))


def geometry_exclusion(L, rings, lines=(), points=(), buffer=0.0, invert=False):
    """(excluded, tie) for one geometry collection (already in the container CRS)."""
    left, top, nx, ny, res = L
    ed, w = ring_edges(rings, orient=True)
    inside = polygon_mask(ed, w, left, res, top, -res, nx, ny, nonzero=True) if len(ed) else np.zeros((ny, nx), bool)
    tie = np.zeros((ny, nx), bool)
    if buffer:
        cx, cy = np.meshgrid(centres(left, res, nx), centres(top, -res, ny))
        d = np.full((ny, nx), np.inf)
        segs = [row for row in ed] + [np.r_[p[k], p[k + 1]] for p in lines for k in range(len(p) - 1)]
        segs += [np.r_[q, q] for p in points for q in p]
        for s in segs:
            d = np.minimum(d, _seg_dist(cx, cy, s))
        b = abs(buffer)
        near = d <= b
        tie = np.abs(d - b) <= TIE * max(1.0, b)
        ex = (inside | near) if buffer > 0 else (inside & ~near)
    else:
        ex = inside
    return (~ex if invert else ex), tie


def shape_availability(rings, crs, res, rasters=(), geometries=()):
    """(eligible, (left, top, nx, ny, res), tie) of one shape: ``rings`` [(ring, is_hole)] in the
    container CRS; ``rasters`` dicts of raster_exclusion's keyword arguments plus ``raster``;
    ``geometries`` dicts of geometry_exclusion's (rings / lines / points in the container CRS)."""
    v = np.concatenate([r for r, _ in rings])
    left, top, nx, ny = window((v[:, 0].min(), v[:, 1].min(), v[:, 0].max(), v[:, 1].max()), res)
    L = (left, top, nx, ny, res)
    ed, w = ring_edges(rings)
    excl = ~polygon_mask(ed, w, left, res, top, -res, nx, ny)
    tie = np.zeros_like(excl)
    for d in rasters:
        ex, t = raster_exclusion(rings, crs, L, **d)
        excl |= ex
        tie |= t
    for d in geometries:
        ex, t = geometry_exclusion(L, **d)
        excl |= ex
        tie |= t
    return ~excl, L, tie


def counts(eligible, L, crs, grid, cutout_crs):
    """(gny, gnx) int64 counts of eligible centres per cutout cell (grid = gx0, gdx, gy0, gdy, gnx,
    gny) and the number of eligible centres within TIE of a cell edge."""
    left, top, nx, ny, res = L
    gx0, gdx, gy0, gdy, gnx, gny = grid
    cx, cy = np.meshgrid(centres(left, res, nx), centres(top, -res, ny))
    px, py = proj.transform(cx[eligible], cy[eligible], crs, cutout_crs)
    u, v = (px - gx0) / gdx, (py - gy0) / gdy
    tie = (np.abs(u - np.round(u)) <= TIE * np.maximum(1, np.abs(u))) | (np.abs(v - np.round(v)) <= TIE * np.maximum(1, np.abs(v)))
    ix, iy = np.floor(u), np.floor(v)
    ok = (ix >= 0) & (ix < gnx) & (iy >= 0) & (iy < gny)
    out = np.zeros((gny, gnx), dtype=np.int64)
    np.add.at(out, (iy[ok].astype(np.int64), ix[ok].astype(np.int64)), 1)
    return out, int(tie.sum()) if crs != cutout_crs else 0
