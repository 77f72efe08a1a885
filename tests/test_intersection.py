"""Intersection matrix (Cutout.intersectionmatrix -> gis.py:148-183): 1.0 where a shape
intersects the closed box of a grid cell.

CPU part: the exact rational checker (oracle/intersection_exact.py) against known
answers, on the dyadic 0.25 degree grid and on the 0.1 degree grid whose float boxes
leave gaps and overlaps; geometry packing.  GPU part: the CUDA kernels
(csrc/indicator.cu, through the C ABI) equal to that checker, with no tolerance.
"""

import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import intersection_exact as IX
import atlite_b200 as ab
from atlite_b200 import gis, synthetic as syn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

X, Y = syn.make_coords(12, 9, 5.0, 40.0)  # 0.25 degree cells: dyadic, the boxes tile exactly
NX = 12


def box(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=float)


def point(x, y):
    return {"type": "Point", "coordinates": [x, y]}


def line(*xy):
    return {"type": "LineString", "coordinates": [list(p) for p in xy]}


def exact(x, y, shapes):
    return IX.intersectionmatrix(x, y, [gis.geometry_parts(s) for s in shapes])


def cells(x, y, shape):
    return {(int(k) // len(x), int(k) % len(x)) for k in np.flatnonzero(exact(x, y, [shape])[0])}


# ------------------------------------------------------------------ oracle known answers (CPU)


def test_kat_cell_touches_its_neighbours():
    """test/test_gis.py:322-332's cell as a shape: the cell and every neighbour sharing its border."""
    for iy, ix, n in ((0, 0, 4), (8, 10, 6), (4, 5, 9)):
        c = box(X[ix] - 0.125, Y[iy] - 0.125, X[ix] + 0.125, Y[iy] + 0.125)
        want = {(j, i) for j in range(iy - 1, iy + 2) for i in range(ix - 1, ix + 2) if 0 <= j < 9 and 0 <= i < NX}
        assert cells(X, Y, c) == want and len(want) == n


def test_points_on_edges_corners_and_inside():
    ex, ey = X[3] + 0.125, Y[4] + 0.125  # the border between columns 3 | 4 and rows 4 | 5
    assert cells(X, Y, point(ex, Y[4])) == {(4, 3), (4, 4)}
    assert cells(X, Y, point(X[3], ey)) == {(4, 3), (5, 3)}
    assert cells(X, Y, point(ex, ey)) == {(4, 3), (4, 4), (5, 3), (5, 4)}
    assert cells(X, Y, point(X[3] + 0.01, Y[4] - 0.02)) == {(4, 3)}
    assert cells(X, Y, point(100.0, 100.0)) == set()


def test_lines_on_borders_and_through_corners():
    yb = Y[2] + 0.125  # row border 2 | 3
    assert cells(X, Y, line((X[1], yb), (X[4], yb))) == {(j, i) for j in (2, 3) for i in range(1, 5)}
    # a diagonal through grid corners touches all four cells at every corner it passes
    c0 = (X[1] - 0.125, Y[1] - 0.125)
    got = cells(X, Y, line(c0, (c0[0] + 0.75, c0[1] + 0.75)))
    want = {(1 + k, 1 + k) for k in range(3)} | {(1 + k, k) for k in range(4)} | {(k, 1 + k) for k in range(4)}
    assert got == want | {(0, 0), (4, 4)}


def test_polygon_with_hole_and_vertex_contact():
    # outer ring: columns 1..6, rows 1..5 (borders exactly on cell edges); hole strictly inside
    # cells (3..4, 3) with a margin, so the cells around the hole's ring are touched and kept,
    # and a cell wholly inside the hole touching no ring is excluded
    outer = box(X[1] - 0.125, Y[1] - 0.125, X[6] + 0.125, Y[5] + 0.125)
    hole = box(X[2] - 0.1, Y[2] - 0.1, X[5] + 0.1, Y[4] + 0.1)[::-1]
    got = cells(X, Y, [outer, hole])
    full = {(j, i) for j in range(0, 7) for i in range(0, 8)}
    assert got == full - {(3, 3), (3, 4)}
    # a triangle that touches cell (6, 6) only at one vertex (its lower-left corner)
    c = (X[6] - 0.125, Y[6] - 0.125)
    tri = np.array([c, (c[0] - 0.1, c[1] - 0.05), (c[0] - 0.05, c[1] - 0.1)])
    assert cells(X, Y, tri) == {(5, 5), (5, 6), (6, 5), (6, 6)}


def test_gaps_and_overlaps_of_the_reference_boxes():
    """0.1 degree cells: box 1 ends at 0.19999999999999998 and box 2 starts at 0.2 (a gap);
    box 5 ends at 0.6000000000000001 and box 6 starts at 0.6 (an overlap)."""
    x, y = syn.make_coords(12, 9, 0.05, 40.05, 0.1, 0.1)
    lo, hi = gis.cell_edges(x)
    assert hi[1] < lo[2] == 0.2 and lo[6] == 0.6 < hi[5]
    assert cells(x, y, point(0.2, y[3])) == {(3, 2)}
    assert cells(x, y, point(0.6, y[3])) == {(3, 5), (3, 6)}
    assert cells(x, y, line((0.2, y[3]), (0.2, y[5]))) == {(3, 2), (4, 2), (5, 2)}


def _clip_meets(a, b, xlo, xhi, ylo, yhi):
    """Closed segment vs closed box by parametric clipping (Liang-Barsky) in rationals:
    an argument independent of orientation signs."""
    from fractions import Fraction as Fr

    t0, t1 = Fr(0), Fr(1)
    for p, q in ((a[0] - b[0], a[0] - xlo), (b[0] - a[0], xhi - a[0]),
                 (a[1] - b[1], a[1] - ylo), (b[1] - a[1], yhi - a[1])):
        if p == 0:
            if q < 0:
                return False
            continue
        t = Fr(q, p)
        if p < 0:
            t0 = max(t0, t)
        else:
            t1 = min(t1, t)
    return t0 <= t1


def test_segment_test_on_near_degenerate_segments():
    """Corner-to-corner segments on the 0.1 and 0.3 degree grids, whose boxes leave gaps and
    overlaps of an ulp, pass within an ulp of other corners: the oracle's separating-axis
    decision from exact orientation signs equals exact parametric clipping."""
    for step in (0.1, 0.3):
        x, y = syn.make_coords(12, 9, 0.05, 40.05, step, step)
        g = IX.Grid(x, y, np.zeros((0, 2)))
        corners = [(g.xlo[i], g.ylo[j]) for j in range(0, 9, 2) for i in range(0, 12, 3)]
        corners += [(g.xhi[i], g.yhi[j]) for j in range(1, 9, 3) for i in range(1, 12, 4)]
        n_hit = 0
        for a in corners:
            for b in corners:
                for j in range(9):
                    for i in range(12):
                        bx = g.box(j, i)
                        hit = IX.segment_meets_box(a, b, *bx)
                        assert hit == _clip_meets(a, b, *bx), (step, a, b, j, i)
                        n_hit += hit
        assert n_hit > 1000


def test_packing_of_every_geometry_kind():
    class Geo:
        def __init__(self, gi):
            self.__geo_interface__ = gi

    ring = box(0, 0, 4, 4)
    closed = np.vstack([ring, ring[:1]]).tolist()
    hole = np.vstack([box(1, 1, 2, 2), box(1, 1, 2, 2)[:1]]).tolist()
    shapes = [
        {"type": "Point", "coordinates": [1.0, 2.0, 3.0]},                          # z dropped
        {"type": "MultiPoint", "coordinates": [[0, 0], [1, 1]]},
        {"type": "LineString", "coordinates": [[0, 0], [1, 0], [1, 1]]},
        {"type": "MultiLineString", "coordinates": [[[0, 0], [1, 0]], [[2, 2], [3, 3], [4, 4]]]},
        Geo({"type": "LinearRing", "coordinates": closed}),
        {"type": "Polygon", "coordinates": [closed, hole]},
        {"type": "MultiPolygon", "coordinates": [[closed], [box(5, 5, 6, 6).tolist()]]},
        {"type": "Feature", "geometry": {"type": "Point", "coordinates": [7, 7]}, "properties": {}},
        {"type": "GeometryCollection", "geometries": [{"type": "Point", "coordinates": [0, 0]},
                                                      {"type": "LineString", "coordinates": [[0, 0], [1, 1]]},
                                                      {"type": "Polygon", "coordinates": [closed]}]},
        None,
        {"type": "Point", "coordinates": []},                                        # empty
        ring,                                                                        # array: a polygon
        [ring, box(1, 1, 2, 2)],
    ]
    spp, pp, kinds, xy = gis.pack_geometries(shapes)
    E, H, L, P = gis.PART_EXTERIOR, gis.PART_HOLE, gis.PART_LINE, gis.PART_POINTS
    per_shape = [kinds[spp[k]:spp[k + 1]].tolist() for k in range(len(shapes))]
    assert per_shape == [[P], [P], [L], [L, L], [L], [E, H], [E, E], [P], [P, L, E], [], [], [E], [E, H]]
    assert np.diff(pp).tolist() == [1, 2, 3, 2, 3, 5, 5, 5, 5, 4, 1, 1, 2, 5, 4, 4, 4]
    assert pp[-1] == len(xy) and xy.dtype == np.float64 and xy.shape[1] == 2
    assert xy[0].tolist() == [1.0, 2.0]
    assert {int(k) for k in (E, H, L, P)} == {0, 1, 2, 3}
    # the polygon readers still reject everything else, with the same error
    with pytest.raises(ValueError, match="unsupported geometry"):
        gis.pack_shapes([{"type": "LineString", "coordinates": [[0, 0], [1, 1]]}])
    with pytest.raises(ValueError, match="unsupported geometry"):
        gis.pack_geometries([{"type": "Curve", "coordinates": []}])
    with pytest.raises(TypeError):
        gis.pack_geometries(["not a geometry"])


def test_intersectionmatrix_requires_the_cutout_crs():
    c = ab.Cutout(data=syn.make_dataset(12, 9, 2, kinds=("temperature",)))
    with pytest.raises(NotImplementedError, match="reprojection"):
        c.intersectionmatrix([point(0.0, 30.0)], shapes_crs=3035)


def test_line_network_generator():
    x, y = syn.make_coords(40, 30, -12.0, 33.0)
    lines = syn.make_line_network(x, y, 25)
    assert len(lines) >= 25 and all(g["type"] == "LineString" for g in lines)
    n = [len(g["coordinates"]) for g in lines]
    assert min(n) >= 2 and max(n) <= 50
    again = syn.make_line_network(x, y, 25)
    assert all((a["coordinates"] == b["coordinates"]).all() for a, b in zip(lines, again))
    kinds = gis.pack_geometries(lines)[2]
    assert (kinds == gis.PART_LINE).all() and len(kinds) == len(lines)


def test_product_does_not_import_the_oracle():
    code = ("import sys, atlite_b200, atlite_b200.gis; "
            "assert 'intersection_exact' not in sys.modules")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=REPO)


# ------------------------------------------------------------------ CUDA kernels (GPU)


def star(rng, cx, cy, r, hole=False):
    k = int(rng.integers(3, 12))
    ang = 2 * np.pi * (np.arange(k) + rng.uniform(0.0, 0.8, k)) / k
    rad = rng.uniform(0.05, 1.0, k) * r
    outer = np.c_[cx + rad * np.cos(ang), cy + 0.7 * rad * np.sin(ang)]
    if not hole:
        return outer
    inner = np.c_[cx + 0.04 * r * np.cos(ang), cy + 0.03 * r * np.sin(ang)][::-1]
    return [outer, inner]


def parity_shapes(x, y, seed):
    """Random and constructed shapes on the grid (x, y)."""
    rng = np.random.default_rng(seed)
    sx, sy = (x[1] - x[0]) / 2, (y[1] - y[0]) / 2
    lo_x, hi_x, lo_y, hi_y = x[0] - sx, x[-1] + sx, y[0] - sy, y[-1] + sy
    span = hi_x - lo_x
    u = lambda: (rng.uniform(lo_x - sx, hi_x + sx), rng.uniform(lo_y - sy, hi_y + sy))  # noqa: E731
    shapes = []
    for t in range(12):
        shapes.append(star(rng, *u(), 0.3 * span, hole=t % 3 == 0))
    for t in range(4):
        a, b = star(rng, *u(), 0.2 * span, hole=True), star(rng, *u(), 0.1 * span)
        shapes.append({"type": "MultiPolygon", "coordinates": [[r.tolist() for r in a], [b.tolist()]]})
    for t in range(10):
        n = int(rng.integers(2, 8))
        shapes.append(line(*[u() for _ in range(n)]))
    # points: random, and on the float box edges and corners
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    pts = [u() for _ in range(20)]
    for _ in range(30):
        i, j = int(rng.integers(len(x))), int(rng.integers(len(y)))
        px = [xlo[i], xhi[i], x[i]][int(rng.integers(3))]
        py = [ylo[j], yhi[j], y[j]][int(rng.integers(3))]
        pts.append((px, py))
    shapes.append({"type": "MultiPoint", "coordinates": [list(p) for p in pts]})
    shapes += [point(*p) for p in pts[20:30]]
    # constructed boundary cases
    shapes += [
        box(xlo[2], ylo[1], xhi[4], yhi[3]),                            # border-aligned box
        line((xlo[1], yhi[2]), (xhi[7], yhi[2])),                        # along a row border
        line((xhi[3], ylo[0]), (xhi[3], yhi[6])),                        # along a column border
        line((xlo[0], ylo[0]), (xhi[5], yhi[5])),                        # corner to corner
        line((xlo[2], yhi[6]), (xhi[8], ylo[0])),                        # anti-diagonal corners
        box(lo_x - 3 * sx, lo_y + sy, lo_x + 3 * sx, lo_y + 5 * sy),     # sticks out on the left
        box(lo_x - 100, lo_y - 100, hi_x + 100, hi_y + 100),             # covers everything
        box(hi_x + 1, hi_y + 1, hi_x + 2, hi_y + 2),                     # outside
        line((hi_x + 1, lo_y), (hi_x + 2, hi_y)),                        # outside
        line((lo_x - 1, y[3]), (hi_x + 1, y[3])),                        # crosses the whole grid
        np.array([[x[4], y[4]]] * 3),                                    # degenerate ring
        line((x[2], y[2]), (x[2], y[2])),                                # zero-length segment
        {"type": "LineString", "coordinates": [[x[5], y[5]]]},           # one-point line
        {"type": "LineString", "coordinates": [[x[1], y[1]], [x[1], y[1]], [x[3], y[2]]]},  # repeated vertex
        {"type": "GeometryCollection", "geometries": []},                # empty
        None,
        {"type": "GeometryCollection", "geometries": [point(x[0], y[0]), line((x[6], y[1]), (x[7], y[4])),
                                                      {"type": "Polygon",
                                                       "coordinates": [box(x[8], y[5], x[9], y[7]).tolist()]}]},
    ]
    return shapes


@pytest.mark.gpu
@pytest.mark.parametrize("step", [0.25, 0.1, 0.3])
def test_gpu_equals_exact_checker(step):
    x, y = syn.make_coords(14, 10, 0.05, 40.05, step, step)
    shapes = parity_shapes(x, y, seed=int(step * 100))
    got = gis.compute_intersectionmatrix(x, y, shapes)
    want = exact(x, y, shapes)
    assert got.shape == want.shape == (len(shapes), 14 * 10)
    assert got.has_sorted_indices and got.indices.dtype == np.int32 and got.dtype == np.float64
    assert (got.data == 1.0).all()
    bad = np.flatnonzero((got.toarray() != want).any(1))
    assert bad.size == 0, f"rows {bad.tolist()} differ"
    assert want[-11].all() and not want[-10].any()  # covers everything; outside


@pytest.mark.gpu
def test_gpu_at_scale_against_indicator_and_checker():
    nx, ny, n = 400, 300, 500
    x, y = syn.make_coords(nx, ny, -12.0, 33.0)
    regions = syn.make_voronoi_shapes(x, y, n)
    lines = syn.make_line_network(x, y, n)
    m = gis.compute_intersectionmatrix(x, y, regions + lines)
    r = m[:n]
    ind = gis.compute_indicatormatrix(x, y, regions)
    assert (ind > 0).multiply(r).nnz == ind.nnz  # the pattern contains the indicator's
    assert (np.asarray(r.sum(0)).ravel() >= 1).all()  # every cell lies in some region
    rng = np.random.default_rng(5)
    pick_r = rng.choice(n, 20, replace=False)
    pick_l = rng.choice(len(lines), 50, replace=False)
    want = IX.intersection_cells(x, y, [gis.geometry_parts(regions[k]) for k in pick_r]
                                 + [gis.geometry_parts(lines[k]) for k in pick_l])
    rows = list(pick_r) + [n + k for k in pick_l]
    for k, w in zip(rows, want):
        assert set(m[k].indices.tolist()) == w, k
    m2 = gis.compute_intersectionmatrix(x, y, regions + lines)
    assert (m.indptr == m2.indptr).all() and (m.indices == m2.indices).all() and (m.data == m2.data).all()
    code = ("import pickle, sys; sys.path.insert(0, %r); "
            "from atlite_b200 import gis, synthetic as syn; "
            "x, y = syn.make_coords(400, 300, -12.0, 33.0); "
            "s = syn.make_voronoi_shapes(x, y, 500) + syn.make_line_network(x, y, 500); "
            "m = gis.compute_intersectionmatrix(x, y, s); "
            "sys.stdout.buffer.write(pickle.dumps((m.indptr, m.indices, m.data)))" % REPO)
    out = subprocess.run([sys.executable, "-c", code], check=True, capture_output=True,
                         env={**os.environ, "ATL_INDICATOR_BUDGET": "2000"}).stdout
    ip, ix, dat = pickle.loads(out)
    assert (ip == m.indptr).all() and (ix == m.indices).all() and (dat == m.data).all()


@pytest.mark.gpu
def test_gpu_cutout_intersectionmatrix_on_a_series_of_mixed_kinds():
    import pandas as pd

    ds = syn.make_dataset(30, 20, 2, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0, kinds=("temperature",))
    c = ab.Cutout(data=ds)
    x, y = np.asarray(c.coords["x"]), np.asarray(c.coords["y"])
    shapes = pd.Series([syn.make_voronoi_shapes(x, y, 3)[0], line((x[0], y[0]), (x[9], y[7])),
                        point(x[4] + 0.25, y[4] + 0.5), None], index=list("abcd"))
    m = c.intersectionmatrix(shapes)
    assert m.shape == (4, 600)
    ref = gis.compute_intersectionmatrix(x, y, list(shapes.values))
    assert (m != ref).nnz == 0
    assert m[2].nnz == 4 and m[3].nnz == 0
