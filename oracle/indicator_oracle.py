"""CPU oracle for the indicator matrix (TEST INFRASTRUCTURE ONLY -- never imported
by atlite_b200; only tests/, __graft_entry__.smoke() and bench.py may use it).

Restates what the reference computes in ``compute_indicatormatrix``
(atlite/gis.py:104-145) for the cells of ``Cutout.grid``
(cutout.py:355-376):  I[i, j] = area(shape_i ∩ cell_j) / area(cell_j).

The reference delegates the geometry to shapely 2.x (GEOS) -- ``d.intersection(o).area``
(gis.py:141-142) -- which is NOT installed in this image and not vendored under
the reference's source tree.  Its algorithm for polygon ∩ axis-aligned box area is restated
here by a DIFFERENT method than the CUDA kernel uses, so the two check each other:
every ring is clipped against the cell rectangle with Sutherland-Hodgman (exact
in area for any simple ring against a convex window) and the shoelace area of the
result is summed, holes negative.  float64, pure Python / NumPy loops: small cases.

PARITY PINNING: **unpinned against shapely** (cannot be executed here).  Pinned
instead on (a) the reference's own known-answer test, test/test_gis.py:322-332
(a shape equal to one grid cell gives exactly 1.0 in that cell and the matrix sums
to 1), restated in tests/test_indicator.py, and (b) analytic areas (rectangles,
triangles, polygon with hole, concave polygon).
"""

from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def _clip_halfplane(poly, axis, bound, keep_greater):
    """Sutherland-Hodgman against one axis-aligned half-plane."""
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
            out.append(r)
    return out


def _shoelace(poly):
    if len(poly) < 3:
        return 0.0
    a = np.asarray(poly, dtype=np.float64)
    x, y = a[:, 0] - a[0, 0], a[:, 1] - a[0, 1]
    return 0.5 * float(np.sum(x * np.roll(y, -1) - np.roll(x, -1) * y))


def ring_cell_area(ring, xlo, xhi, ylo, yhi):
    """|area| of ring ∩ [xlo, xhi] x [ylo, yhi]."""
    poly = [list(map(float, p[:2])) for p in ring]
    if len(poly) > 1 and poly[0] == poly[-1]:
        poly = poly[:-1]
    for axis, bound, greater in ((0, xlo, True), (0, xhi, False), (1, ylo, True), (1, yhi, False)):
        poly = _clip_halfplane(poly, axis, bound, greater)
        if len(poly) < 3:
            return 0.0
    return abs(_shoelace(poly))


def indicatormatrix(x, y, shapes, keep=1e-10):
    """shapes: list of shapes, each a list of (ring (N,2), is_hole) -- the output of
    atlite_b200.gis.geometry_rings.  Returns CSR (n_shapes, ny*nx)."""
    x, y = np.asarray(x, float), np.asarray(y, float)
    dx, dy = (x[-1] - x[0]) / (len(x) - 1), (y[-1] - y[0]) / (len(y) - 1)
    nx, ny = len(x), len(y)
    rows, cols, vals = [], [], []
    for i, rings in enumerate(shapes):
        acc = {}
        for ring, hole in rings:
            r = np.asarray(ring, float)
            if len(r) < 3:
                continue
            i0 = max(int(np.floor((r[:, 0].min() - (x[0] - dx / 2)) / dx)), 0)
            i1 = min(int(np.ceil((r[:, 0].max() - (x[0] - dx / 2)) / dx)), nx)
            j0 = max(int(np.floor((r[:, 1].min() - (y[0] - dy / 2)) / dy)), 0)
            j1 = min(int(np.ceil((r[:, 1].max() - (y[0] - dy / 2)) / dy)), ny)
            for j in range(j0, j1):
                for k in range(i0, i1):
                    a = ring_cell_area(r, x[k] - dx / 2, x[k] + dx / 2, y[j] - dy / 2, y[j] + dy / 2)
                    if a:
                        acc[j * nx + k] = acc.get(j * nx + k, 0.0) + (-a if hole else a)
        for c in sorted(acc):
            f = acc[c] / (dx * dy)
            if f > keep:
                rows.append(i)
                cols.append(c)
                vals.append(min(f, 1.0))
    return sp.csr_matrix((vals, (rows, cols)), shape=(len(shapes), ny * nx))
