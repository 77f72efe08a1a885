"""EXACT checker for the intersection matrix (TEST INFRASTRUCTURE ONLY).

The reference's ``compute_intersectionmatrix`` (atlite/gis.py:148-183) sets
I[i, j] = 1 when ``cell_j.intersects(shape_i)`` in shapely / GEOS, with the cells of
``Cutout.grid`` (cutout.py:369-372): box(x - sx, y - sy, x + sx, y + sy) in float64,
(sx, sy) = (x[1] - x[0], y[1] - y[0]) / 2.  Shapely cannot run in this image, so this
module is the reference: the same closed-set predicate in exact rational arithmetic.

  * The float64 boxes are built as the reference builds them and converted exactly,
    together with every vertex, to integers over one common power-of-two denominator,
    so every test below is integer arithmetic with no rounding at all.
  * Point vs box: closed comparisons.
  * Segment vs closed box: separating axes -- the box axes (bounding boxes) and the
    segment's normal (all four corners strictly on one side of its line).
  * Polygon: the cells some ring edge touches, plus the cells wholly inside the
    polygon; a cell no ring edge touches is wholly inside or outside, and its centre
    decides, by the even-odd rule over the polygon's exterior and holes.

A shape is a list of (kind, (N, 2) coordinates) parts as ``gis.geometry_parts`` yields
them; a hole belongs to the exterior before it.  Pure Python: small cases only.
"""

from __future__ import annotations

import bisect
from fractions import Fraction as Fr

import numpy as np

EXTERIOR, HOLE, LINE, POINTS = 0, 1, 2, 3


def orient(a, b, c):
    """Exact orient2d: > 0 when c lies left of the line a -> b."""
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def segment_meets_box(a, b, xlo, xhi, ylo, yhi):
    """Closed segment [a, b] vs closed box, by separating axes (a == b: a point)."""
    if max(a[0], b[0]) < xlo or min(a[0], b[0]) > xhi or max(a[1], b[1]) < ylo or min(a[1], b[1]) > yhi:
        return False
    s = [orient(a, b, c) for c in ((xlo, ylo), (xhi, ylo), (xhi, yhi), (xlo, yhi))]
    return not (all(v > 0 for v in s) or all(v < 0 for v in s))


class Grid:
    """The reference boxes of a cutout grid as integers over a common denominator."""

    def __init__(self, x, y, vertices):
        nx = len(x)
        xs, ys = np.meshgrid(np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64))
        coords = np.asarray((np.ravel(xs), np.ravel(ys))).T  # cutout.py:369-371, as written there
        span = (coords[nx + 1] - coords[0]) / 2
        lo, hi = coords - span, coords + span
        xlo, xhi, ylo, yhi = lo[:nx, 0], hi[:nx, 0], lo[::nx, 1], hi[::nx, 1]
        floats = np.concatenate([xlo, xhi, ylo, yhi, np.asarray(vertices, dtype=np.float64).ravel()])
        self.den = max(Fr(float(v)).denominator for v in floats)  # powers of two: the largest is the lcm
        self.xlo, self.xhi = [self.int(v) for v in xlo], [self.int(v) for v in xhi]
        self.ylo, self.yhi = [self.int(v) for v in ylo], [self.int(v) for v in yhi]
        self.nx, self.ny = len(xlo), len(ylo)

    def int(self, v):
        f = Fr(float(v)) * self.den
        assert f.denominator == 1
        return f.numerator

    def cells_overlapping(self, x0, x1, y0, y1):
        """(iy, ix) of every box meeting the closed rectangle [x0, x1] x [y0, y1]."""
        # boxes are ordered: xlo and xhi non-decreasing
        i0 = bisect.bisect_left(self.xhi, x0)
        i1 = bisect.bisect_right(self.xlo, x1)
        j0 = bisect.bisect_left(self.yhi, y0)
        j1 = bisect.bisect_right(self.ylo, y1)
        return [(j, i) for j in range(j0, j1) for i in range(i0, i1)]

    def box(self, j, i):
        return self.xlo[i], self.xhi[i], self.ylo[j], self.yhi[j]


def _segments(kind, pts):
    if kind == POINTS or len(pts) == 1:
        return [(p, p) for p in pts]
    if kind == LINE:
        return list(zip(pts[:-1], pts[1:]))
    return list(zip(pts, pts[1:] + pts[:1]))  # ring: the closing edge included


def _inside(rings, cx2, cy2):
    """Even-odd rule for the point (cx2 / 2, cy2 / 2) against the rings (integer vertices)."""
    odd = False
    for r in rings:
        for (px, py), (qx, qy) in zip(r, r[1:] + r[:1]):
            px, py, qx, qy = 2 * px, 2 * py, 2 * qx, 2 * qy
            if (py > cy2) != (qy > cy2):
                # crossing x of the edge at cy2, compared with cx2 without division
                lhs, rhs = (cx2 - px) * (qy - py), (cy2 - py) * (qx - px)
                if (lhs < rhs) if qy > py else (lhs > rhs):
                    odd = not odd
    return odd


def shape_cells(grid, parts):
    """Set of flat cell indices (iy * nx + ix) the shape intersects."""
    hit = set()
    polygons = []  # [[exterior, hole, ...], ...] with integer vertices
    for kind, coords in parts:
        pts = [(grid.int(p[0]), grid.int(p[1])) for p in np.asarray(coords, dtype=np.float64)[:, :2]]
        if not pts:
            continue
        if kind == EXTERIOR:
            polygons.append([pts])
        elif kind == HOLE:
            polygons[-1].append(pts)
        for a, b in _segments(kind, pts):
            for j, i in grid.cells_overlapping(min(a[0], b[0]), max(a[0], b[0]), min(a[1], b[1]), max(a[1], b[1])):
                if (j, i) not in hit and segment_meets_box(a, b, *grid.box(j, i)):
                    hit.add((j, i))
    for rings in polygons:
        ext = rings[0]
        xs, ys = [p[0] for p in ext], [p[1] for p in ext]
        for j, i in grid.cells_overlapping(min(xs), max(xs), min(ys), max(ys)):
            if (j, i) in hit:
                continue
            xlo, xhi, ylo, yhi = grid.box(j, i)
            if _inside(rings, xlo + xhi, ylo + yhi):
                hit.add((j, i))
    return {j * grid.nx + i for j, i in hit}


def intersection_cells(x, y, shapes):
    """[set of flat cell indices] per shape; ``shapes`` = lists of (kind, coords) parts."""
    verts = [np.asarray(c, dtype=np.float64)[:, :2] for parts in shapes for _, c in parts if len(c)]
    grid = Grid(x, y, np.concatenate(verts) if verts else np.zeros((0, 2)))
    return [shape_cells(grid, parts) for parts in shapes]


def intersectionmatrix(x, y, shapes):
    """Dense (n_shapes, ny * nx) float64 0/1 matrix."""
    cells = intersection_cells(x, y, shapes)
    out = np.zeros((len(shapes), len(x) * len(y)))
    for k, c in enumerate(cells):
        out[k, sorted(c)] = 1.0
    return out
