"""EXACT second checker for the indicator matrix (TEST INFRASTRUCTURE ONLY).

``oracle/indicator_oracle.py`` restates ``compute_indicatormatrix``
(atlite/gis.py:104-145: I[i, j] = area(shape_i ∩ cell_j) / area(cell_j)) in
float64; shapely / GEOS, which the reference delegates to, cannot run in this image.  This
module removes floating point from the question: the same quantity in exact rational
arithmetic (``fractions.Fraction``; every float64 input converts exactly), so the float
oracle and the CUDA kernels are both measured against numbers that carry no rounding at
all.  Method: every ring is clipped against the four half-planes of the cell
(Sutherland-Hodgman; exact for a simple ring against a convex window when the intersection
points are exact, which they are here) and the shoelace sum of the clipped ring is taken,
holes negative.  Cell edges are x[k] -/+ dx/2 with dx = (x[-1] - x[0]) / (nx - 1), all
rational.  Pure Python: tiny cases only.
"""

from __future__ import annotations

from fractions import Fraction as Fr


def _clip(poly, axis, bound, keep_greater):
    out = []
    n = len(poly)
    for k in range(n):
        p, q = poly[k], poly[(k + 1) % n]
        pin = (p[axis] >= bound) if keep_greater else (p[axis] <= bound)
        qin = (q[axis] >= bound) if keep_greater else (q[axis] <= bound)
        if pin:
            out.append(p)
        if pin != qin:
            t = (bound - p[axis]) / (q[axis] - p[axis])
            r = [p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1])]
            r[axis] = bound
            out.append(tuple(r))
    return out


def _area2(poly):
    """Twice the signed shoelace area."""
    return sum(poly[k][0] * poly[(k + 1) % len(poly)][1] - poly[(k + 1) % len(poly)][0] * poly[k][1]
               for k in range(len(poly)))


def ring_cell_area(ring, xlo, xhi, ylo, yhi):
    poly = [(Fr(float(p[0])), Fr(float(p[1]))) for p in ring]
    if len(poly) > 1 and poly[0] == poly[-1]:
        poly = poly[:-1]
    for axis, bound, greater in ((0, xlo, True), (0, xhi, False), (1, ylo, True), (1, yhi, False)):
        poly = _clip(poly, axis, bound, greater)
        if len(poly) < 3:
            return Fr(0)
    return abs(_area2(poly)) / 2


def indicator_fractions(x, y, shapes):
    """{(shape, cell): Fraction of the cell covered}, cells in cutout.grid order
    (iy * nx + ix), only non-zero entries.  ``shapes`` as for indicator_oracle.indicatormatrix."""
    fx, fy = [Fr(float(v)) for v in x], [Fr(float(v)) for v in y]
    nx, ny = len(fx), len(fy)
    dx, dy = (fx[-1] - fx[0]) / (nx - 1), (fy[-1] - fy[0]) / (ny - 1)
    out = {}
    for i, rings in enumerate(shapes):
        for ring, hole in rings:
            if len(ring) < 3:
                continue
            xs, ys = [Fr(float(p[0])) for p in ring], [Fr(float(p[1])) for p in ring]
            for j in range(ny):
                ylo, yhi = fy[j] - dy / 2, fy[j] + dy / 2
                if max(ys) <= ylo or min(ys) >= yhi:
                    continue
                for k in range(nx):
                    xlo, xhi = fx[k] - dx / 2, fx[k] + dx / 2
                    if max(xs) <= xlo or min(xs) >= xhi:
                        continue
                    a = ring_cell_area(ring, xlo, xhi, ylo, yhi)
                    if a:
                        key = (i, j * nx + k)
                        out[key] = out.get(key, Fr(0)) + (-a if hole else a) / (dx * dy)
    return {k: v for k, v in out.items() if v != 0}
