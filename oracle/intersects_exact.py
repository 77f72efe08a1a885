"""EXACT checker for the general form of the intersection matrix (TEST INFRASTRUCTURE ONLY).

The reference's ``compute_intersectionmatrix(orig, dest)`` (atlite/gis.py:148-183) sets
I[i, j] = 1 when ``orig_j.intersects(dest_i)`` in shapely / GEOS: the two closed point sets share a
point.  Shapely cannot run in this image, so this module is the reference, in exact arithmetic.

Point set of a shape (a list of (kind, (N, 2) coordinates) parts as ``gis.geometry_parts`` yields
them), the one ``intersection_exact`` uses for a shape against a cell:
  * every segment of every part: ring edges with the closing edge, line segments, and points as
    zero-length segments;
  * the even-odd interior of each polygon, an exterior together with the holes that follow it (a
    hole before any exterior of its shape is a polygon of its own); a shape is the union of its
    polygons.

Two shapes intersect when a segment of one meets a segment of the other (orientation signs, and
the overlap of the 1-D projections of collinear segments), or else when some part of one lies
inside a polygon of the other.  With no segment in common, every connected part (a ring, a line,
one point) lies wholly inside or wholly outside each polygon of the other shape, so its first
vertex decides, by the even-odd rule with a half-open crossing rule.

Every float64 is converted to a ``Fraction`` exactly, so every sign is exact.  NumPy only narrows
the candidates: float comparisons of coordinates are exact too.
"""

from __future__ import annotations

from fractions import Fraction as Fr

import numpy as np

EXTERIOR, HOLE, LINE, POINTS = 0, 1, 2, 3


def orient(a, b, c):
    """Exact orient2d of Fractions: > 0 when c lies left of the line a -> b."""
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def _sign(v):
    return (v > 0) - (v < 0)


def segments_meet(a, b, c, d):
    """Closed segments [a, b] and [c, d] (a == b or c == d: a point) share a point."""
    if (max(a[0], b[0]) < min(c[0], d[0]) or min(a[0], b[0]) > max(c[0], d[0]) or
            max(a[1], b[1]) < min(c[1], d[1]) or min(a[1], b[1]) > max(c[1], d[1])):
        return False
    if a == b:
        return c == d or orient(c, d, a) == 0
    if c == d:
        return orient(a, b, c) == 0
    if _sign(orient(a, b, c)) * _sign(orient(a, b, d)) > 0:
        return False
    return _sign(orient(c, d, a)) * _sign(orient(c, d, b)) <= 0  # collinear: the boxes overlap


class Shape:
    """Segments (float array and exact endpoints), polygon of each ring segment, probes, box."""

    def __init__(self, parts):
        seg, poly, probes = [], [], []
        n_poly, cur = 0, -1
        for kind, coords in parts:
            pts = [tuple(map(float, p[:2])) for p in np.asarray(coords, dtype=np.float64)]
            if not pts:
                continue
            if kind == POINTS:
                seg += [(p, p) for p in pts]
                poly += [-1] * len(pts)
                probes += pts
                continue
            probes.append(pts[0])
            if kind == LINE:
                s = [(pts[0], pts[0])] if len(pts) == 1 else list(zip(pts[:-1], pts[1:]))
                seg += s
                poly += [-1] * len(s)
                continue
            if kind == EXTERIOR or cur < 0:
                cur, n_poly = n_poly, n_poly + 1
            seg += list(zip(pts, pts[1:] + pts[:1]))
            poly += [cur] * len(pts)
        self.seg = np.array([[a[0], a[1], b[0], b[1]] for a, b in seg], dtype=np.float64).reshape(-1, 4)
        self.poly = np.array(poly, dtype=np.int64)
        self.probes = probes
        self.empty = len(seg) == 0
        if not self.empty:
            s = self.seg
            self.box = (min(s[:, 0].min(), s[:, 2].min()), min(s[:, 1].min(), s[:, 3].min()),
                        max(s[:, 0].max(), s[:, 2].max()), max(s[:, 1].max(), s[:, 3].max()))

    def exact(self, k):
        ax, ay, bx, by = self.seg[k]
        return (Fr(ax), Fr(ay)), (Fr(bx), Fr(by))

    def near(self, xlo, ylo, xhi, yhi):
        """Indices of the segments whose boxes meet the closed box."""
        s = self.seg
        return np.flatnonzero((np.maximum(s[:, 0], s[:, 2]) >= xlo) & (np.minimum(s[:, 0], s[:, 2]) <= xhi) &
                              (np.maximum(s[:, 1], s[:, 3]) >= ylo) & (np.minimum(s[:, 1], s[:, 3]) <= yhi))

    def inside(self, p):
        """p (on no segment of the shape) lies inside one of its polygons: even-odd per polygon."""
        s, py = self.seg, p[1]
        span = np.flatnonzero((self.poly >= 0) & ((s[:, 1] > py) != (s[:, 3] > py)))
        q = (Fr(p[0]), Fr(p[1]))
        odd = {}
        for k in span:
            a, b = self.exact(k)
            o = orient(a, b, q)
            if (o > 0) if b[1] > a[1] else (o < 0):  # the crossing lies right of p
                odd[self.poly[k]] = not odd.get(self.poly[k], False)
        return any(odd.values())


def _boxes_meet(a, b):
    return a[0] <= b[2] and b[0] <= a[2] and a[1] <= b[3] and b[1] <= a[3]


def shapes_intersect(A, B):
    """Closed point sets of the ``Shape``s A and B share a point."""
    if A.empty or B.empty or not _boxes_meet(A.box, B.box):
        return False
    for i in A.near(*B.box):
        a, b = A.exact(i)
        ax, ay, bx, by = A.seg[i]
        for j in B.near(min(ax, bx), min(ay, by), max(ax, bx), max(ay, by)):
            if segments_meet(a, b, *B.exact(j)):
                return True
    for S, T in ((A, B), (B, A)):
        for p in S.probes:
            if T.box[0] <= p[0] <= T.box[2] and T.box[1] <= p[1] <= T.box[3] and T.inside(p):
                return True
    return False


def intersects(parts_a, parts_b):
    """Two shapes given as (kind, coords) part lists intersect."""
    return shapes_intersect(Shape(parts_a), Shape(parts_b))


def intersects_pairs(orig, dest):
    """{(i, j)}: dest_i intersects orig_j; ``orig`` and ``dest`` are lists of part lists."""
    O, D = [Shape(p) for p in orig], [Shape(p) for p in dest]
    ob = np.array([o.box if not o.empty else (np.inf, np.inf, -np.inf, -np.inf) for o in O]).reshape(-1, 4)
    out = set()
    for i, d in enumerate(D):
        if d.empty:
            continue
        near = np.flatnonzero((ob[:, 0] <= d.box[2]) & (d.box[0] <= ob[:, 2]) &
                              (ob[:, 1] <= d.box[3]) & (d.box[1] <= ob[:, 3]))
        out |= {(i, int(j)) for j in near if shapes_intersect(d, O[j])}
    return out


def intersects_matrix(orig, dest):
    """Dense (len(dest), len(orig)) float64 0/1 matrix."""
    out = np.zeros((len(dest), len(orig)))
    for i, j in intersects_pairs(orig, dest):
        out[i, j] = 1.0
    return out
