"""Indicator matrix (SURVEY section 8 f1): shapes -> covered cell fractions.

CPU part: the Sutherland-Hodgman oracle against known answers -- the reference's own
known-answer test (test/test_gis.py:322-332: a shape equal to one grid cell) and
analytic areas -- plus the host-side shape packing and the C entry points' input checks.  GPU part: the CUDA
edge-accumulation kernels (csrc/indicator.cu, through the C ABI) against that oracle
and through size-independent properties at scale.
"""

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import indicator_oracle as IO
import atlite_b200 as ab
from atlite_b200 import _lib, gis, synthetic as syn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def box(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=float)


def oracle(x, y, shapes):
    return IO.indicatormatrix(x, y, [gis.geometry_rings(s) for s in shapes])


def shoelace(ring):
    r = np.asarray(ring, float)
    return 0.5 * abs(np.sum(r[:, 0] * np.roll(r[:, 1], -1) - np.roll(r[:, 0], -1) * r[:, 1]))


X, Y = syn.make_coords(12, 9, 5.0, 40.0)  # 0.25 degree cells


# ------------------------------------------------------------------ oracle known answers (CPU)


def test_oracle_reference_kat_cell_shape_gives_exactly_one():
    """test/test_gis.py:322-332: indicatormatrix([cell]) has a single 1.0."""
    for iy, ix in ((0, 0), (8, 10)):  # lower-left cell; the reference's `iloc[-2]`
        cell = box(X[ix] - 0.125, Y[iy] - 0.125, X[ix] + 0.125, Y[iy] + 0.125)
        m = oracle(X, Y, [cell])
        assert m[0, iy * 12 + ix] == 1.0
        assert m.sum() == 1


def test_oracle_analytic_areas():
    # a box covering 2.5 x 1.5 cells, offset by half a cell
    b = box(X[2], Y[3], X[2] + 2.5 * 0.25, Y[3] + 1.5 * 0.25)
    m = oracle(X, Y, [b]).toarray().reshape(9, 12)
    assert np.isclose(m.sum(), 2.5 * 1.5)
    np.testing.assert_allclose(m[3, 2:5], [0.25, 0.5, 0.5])
    # triangle with legs of 2 cells: area 2 cells, the hypotenuse halves the diagonal cells
    x, y = np.arange(4.0), np.arange(3.0)
    t = np.array([[-0.5, -0.5], [1.5, -0.5], [-0.5, 1.5]])
    m = oracle(x, y, [t]).toarray().reshape(3, 4)
    np.testing.assert_allclose(m, [[1, 0.5, 0, 0], [0.5, 0, 0, 0], [0, 0, 0, 0]])
    # polygon with a hole, both orientations of both rings: same answer
    outer, hole = box(-0.5, -0.5, 2.5, 1.5), box(0.5, -0.25, 1.5, 0.75)
    for o in (outer, outer[::-1]):
        for h in (hole, hole[::-1]):
            m = oracle(x, y, [[o, h]]).toarray().reshape(3, 4)
            assert np.isclose(m.sum(), 6 - 1)
            assert np.isclose(m[0, 1], 1 - 0.75) and np.isclose(m[1, 1], 1 - 0.25)
    # concave (L-shaped) polygon: area 3 cells
    L = np.array([[-0.5, -0.5], [1.5, -0.5], [1.5, 0.5], [0.5, 0.5], [0.5, 1.5], [-0.5, 1.5]])
    m = oracle(x, y, [L]).toarray().reshape(3, 4)
    np.testing.assert_allclose(m, [[1, 1, 0, 0], [1, 0, 0, 0], [0, 0, 0, 0]])


def _random_polygon(rng, cx, cy, r, n, hole=False):
    """Star-shaped (hence simple) polygon around (cx, cy); optionally with a hole."""
    ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    rad = rng.uniform(0.45 * r, r, n)
    outer = np.c_[cx + rad * np.cos(ang), cy + rad * np.sin(ang)]
    if not hole:
        return outer
    a2 = np.sort(rng.uniform(0, 2 * np.pi, 5))
    inner = np.c_[cx + 0.3 * r * np.cos(a2), cy + 0.3 * r * np.sin(a2)]
    return [outer, inner[::-1]]


def test_float_oracle_against_exact_rational_arithmetic():
    """The float64 oracle against the SAME quantity in exact rational arithmetic
    (oracle/indicator_exact.py): no rounding on the checker's side, so the bound below is the
    float oracle's own arithmetic error (shapely cannot run in this image)."""
    import indicator_exact as IE

    rng = np.random.default_rng(11)
    x, y = syn.make_coords(9, 7, -1.0, 50.0, 0.5, 0.25)
    shapes = [_random_polygon(rng, 0.8, 50.6, 1.3, 9), _random_polygon(rng, 1.9, 50.9, 0.9, 7, hole=True),
              box(x[2] - 0.25, y[1] - 0.125, x[4] + 0.25, y[3] + 0.125),  # edges exactly on cell borders
              _random_polygon(rng, -1.4, 49.9, 1.0, 6),                   # sticks out of the grid
              np.array([[0.1, 50.1], [2.3, 50.15], [0.1, 50.2]])]          # sliver
    rings = [gis.geometry_rings(s) for s in shapes]
    exact = IE.indicator_fractions(x, y, rings)
    m = IO.indicatormatrix(x, y, rings, keep=0.0).tocoo()
    got = {(int(i), int(j)): v for i, j, v in zip(m.row, m.col, m.data)}
    assert set(got) == set(exact)
    worst = max(abs(got[k] - float(exact[k])) for k in exact)
    assert worst < 1e-13, worst  # observed 1.7e-14 (coordinates ~50, cells 0.25: shoelace cancellation)
    # exact partition facts: the border-aligned box covers exactly 3 x 3 whole cells
    box_cells = {k: v for k, v in exact.items() if k[0] == 2}
    assert len(box_cells) == 9 and all(v == 1 for v in box_cells.values())
    # the hole is subtracted exactly: total == area(outer) - area(inner) in cell units
    import fractions

    def area(r):
        pts = [(fractions.Fraction(float(a)), fractions.Fraction(float(b))) for a, b in r]
        return abs(sum(pts[k][0] * pts[(k + 1) % len(pts)][1] - pts[(k + 1) % len(pts)][0] * pts[k][1]
                       for k in range(len(pts)))) / 2

    cell = fractions.Fraction(1, 2) * fractions.Fraction(1, 4)
    total = sum(v for k, v in exact.items() if k[0] == 1)
    assert total == (area(shapes[1][0]) - area(shapes[1][1])) / cell  # the polygon lies inside the grid


def test_exact_checker_reference_kat():
    """test/test_gis.py:322-332 in exact arithmetic: the first grid cell and the
    reference's `iloc[-2]` cell as shapes -> exactly one entry, exactly 1."""
    import indicator_exact as IE

    for iy, ix in ((0, 0), (8, 10)):
        cell = box(X[ix] - 0.125, Y[iy] - 0.125, X[ix] + 0.125, Y[iy] + 0.125)
        ex = IE.indicator_fractions(X, Y, [gis.geometry_rings(cell)])
        assert ex == {(0, iy * 12 + ix): 1}


def test_shape_packing_accepts_geojson_geo_interface_and_arrays():
    ring, hole = box(0, 0, 4, 4), box(1, 1, 2, 2)

    class Geo:  # what shapely / geopandas objects expose
        def __init__(self, gi):
            self.__geo_interface__ = gi

    closed = np.vstack([ring, ring[:1]])
    poly = {"type": "Polygon", "coordinates": [closed.tolist(), np.vstack([hole, hole[:1]]).tolist()]}
    multi = {"type": "MultiPolygon", "coordinates": [[closed.tolist()], [box(5, 5, 6, 6).tolist()]]}
    feature = {"type": "Feature", "geometry": poly, "properties": {}}
    srp, rp, holes, xy = gis.pack_shapes([ring, [ring, hole], poly, Geo(multi), feature, None])
    assert srp.tolist() == [0, 1, 3, 5, 7, 9, 9]
    assert holes.tolist() == [0, 0, 1, 0, 1, 0, 0, 0, 1]
    assert rp[-1] == len(xy) and xy.dtype == np.float64 and xy.shape[1] == 2
    # collections: dict and pandas Series keep their order
    import pandas as pd

    a = gis.pack_shapes({"a": ring, "b": [ring, hole]})
    b = gis.pack_shapes(pd.Series([ring, [ring, hole]], index=["a", "b"]))
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u, v)
    with pytest.raises(ValueError, match="unsupported geometry"):
        gis.pack_shapes([{"type": "Point", "coordinates": [0, 0]}])
    with pytest.raises(TypeError):
        gis.pack_shapes(["not a polygon"])


def test_c_entries_check_every_ring_before_device_work():
    """atl_indicator_compute and atl_intersection_compute refuse a malformed shape with the input
    error before they select the device, so the error is the same with or without a usable GPU."""
    lib = _lib.load()
    x, y = np.arange(4.0), np.arange(3.0)
    edges = [*gis.cell_edges(x), *gis.cell_edges(y)]
    srp, rp, kinds, xy = gis.pack_shapes([box(0.2, 0.2, 1.8, 1.8), box(1.2, 0.2, 2.8, 1.8)])
    bad_xy = xy.copy()
    bad_xy[5, 1] = np.nan
    cases = [((np.array([0, 1, 0], dtype=np.int64), rp, xy), "shape_{}_ptr must be non-decreasing"),
             ((srp, np.array([0, 4, 2], dtype=np.int64), xy), "{}_ptr must be non-decreasing"),
             ((srp, rp, bad_xy), "non-finite vertex")]
    h = C.c_void_p()
    for (s, r, v), msg in cases:
        shapes = [_lib.ptr(a) for a in (s, r, kinds, v)]
        rc = lib.atl_indicator_compute(0, 3, 4, 0.0, 1.0, 0.0, 1.0, 2, *shapes, C.byref(h))
        assert rc == -1 and not h.value
        assert msg.format("ring").encode() in lib.atl_last_error()
        rc = lib.atl_intersection_compute(0, 3, 4, 0.0, 1.0, 0.0, 1.0, *map(_lib.ptr, edges), 2, *shapes, C.byref(h))
        assert rc == -1 and not h.value
        assert msg.format("part").encode() in lib.atl_last_error()


def test_grid_axis_validation():
    assert gis.regular_axis([1.0, 1.25, 1.5], "x") == (1.0, 0.25)
    for bad in ([1.0], [3.0, 2.0, 1.0], [0.0, 1.0, 3.0]):
        with pytest.raises(ValueError):
            gis.regular_axis(bad, "x")
    c = ab.Cutout(data=syn.make_dataset(12, 9, 2, kinds=("temperature",)))
    with pytest.raises(NotImplementedError, match="reprojection"):
        c.indicatormatrix([box(0, 0, 1, 1)], shapes_crs=3035)


def test_product_does_not_import_the_oracle():
    code = ("import sys, atlite_b200, atlite_b200.gis; "
            "assert 'indicator_oracle' not in sys.modules and 'atlite_oracle' not in sys.modules")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=REPO)


# ------------------------------------------------------------------ CUDA kernels (GPU)


def random_shapes(rng, n, x, y):
    shapes = []
    for t in range(n):
        k = rng.integers(3, 12)
        # one vertex per angular sector: gaps stay below pi, so the ring is star-shaped
        # about c and therefore simple (invalid rings have no defined overlap area)
        ang = 2 * np.pi * (np.arange(k) + rng.uniform(0.0, 0.8, k)) / k
        rad = rng.uniform(0.05, 1.2, k)
        c = np.array([rng.uniform(x[0] - 0.5, x[-1] + 0.5), rng.uniform(y[0] - 0.5, y[-1] + 0.5)])
        ring = np.c_[c[0] + rad * np.cos(ang), c[1] + 0.6 * rad * np.sin(ang)]  # star-shaped, maybe concave
        if t % 2:
            ring = ring[::-1]
        rings = [ring]
        if t % 3 == 0:  # a hole strictly inside
            rings.append(np.c_[c[0] + 0.02 * np.cos(ang), c[1] + 0.012 * np.sin(ang)])
        if t % 5 == 0:  # second part: MultiPolygon as GeoJSON
            far = box(x[0] + 0.3, y[0] + 0.1, x[0] + 0.9, y[0] + 0.45)
            shapes.append({"type": "MultiPolygon",
                           "coordinates": [[np.vstack([r, r[:1]]).tolist() for r in rings],
                                           [np.vstack([far, far[:1]]).tolist()]]})
        else:
            shapes.append(rings)
    return shapes


@pytest.mark.gpu
def test_gpu_matches_oracle_on_random_polygons():
    rng = np.random.default_rng(11)
    shapes = random_shapes(rng, 40, X, Y)
    shapes += [box(X[0] - 0.125, Y[0] - 0.125, X[0] + 0.125, Y[0] + 0.125),   # the reference KAT
               box(-50, -50, 80, 80),                                      # covers everything
               box(100, 100, 101, 101),                                    # entirely outside
               box(X[3], Y[0] - 3, X[5], Y[0] + 0.01),                      # sticks out below
               np.array([[6.0, 41.0], [6.0, 41.0], [6.0, 41.0]]),           # degenerate
               np.array([[6.0, 41.0], [7.0, 41.0]])]                        # two points
    got = gis.compute_indicatormatrix(X, Y, shapes)
    want = oracle(X, Y, shapes)
    assert got.shape == want.shape == (len(shapes), 9 * 12)
    assert got.has_sorted_indices and got.indices.dtype == np.int32
    np.testing.assert_allclose(got.toarray(), want.toarray(), rtol=0, atol=2e-12)
    assert got[40, 0] == 1.0 and got[40].sum() == 1           # exactly, like test_gis.py:322-332
    assert got[41].nnz == 108 and (got[41].data == 1.0).all()
    assert got[42].nnz == got[44].nnz == got[45].nnz == 0
    # same sparsity pattern as the oracle wherever the value is not at the keep threshold
    w = want.toarray()
    assert ((got.toarray() > 0) == (w > 0))[np.abs(w - 1e-10) > 1e-11].all()


@pytest.mark.gpu
def test_gpu_matches_exact_rational_arithmetic():
    """The CUDA kernels against exact rational areas (no float oracle in between)."""
    import indicator_exact as IE

    rng = np.random.default_rng(12)
    x, y = syn.make_coords(9, 7, -1.0, 50.0, 0.5, 0.25)
    shapes = [_random_polygon(rng, 0.8, 50.6, 1.3, 11), _random_polygon(rng, 1.9, 50.9, 0.9, 8, hole=True),
              box(x[2] - 0.25, y[1] - 0.125, x[4] + 0.25, y[3] + 0.125),
              _random_polygon(rng, -1.4, 49.9, 1.0, 6)]
    exact = IE.indicator_fractions(x, y, [gis.geometry_rings(s) for s in shapes])
    m = gis.compute_indicatormatrix(x, y, shapes).tocoo()
    got = {(int(i), int(j)): v for i, j, v in zip(m.row, m.col, m.data)}
    big = {k for k, v in exact.items() if v > 1e-9}
    assert big <= set(got)
    assert max(abs(got[k] - float(exact[k])) for k in big) < 2e-12
    assert all(float(exact.get(k, 0)) < 1e-9 or k in big for k in got)
    for k, v in got.items():
        if k[0] == 2:
            assert v == 1.0  # border-aligned box: exactly whole cells


@pytest.mark.gpu
def test_gpu_partition_of_unity_and_areas_at_scale():
    """Voronoi regions partition the extent: every cell's column sums to 1, every
    row sums to the polygon's area in cells; bit-identical run to run; batching."""
    nx, ny, n = 400, 300, 500
    x, y = syn.make_coords(nx, ny, -12.0, 33.0)
    rings = syn.make_voronoi_shapes(x, y, n)
    m = gis.compute_indicatormatrix(x, y, rings)
    np.testing.assert_allclose(np.asarray(m.sum(0)).ravel(), 1.0, rtol=0, atol=1e-9)
    area = np.array([shoelace(r) for r in rings]) / 0.25**2
    np.testing.assert_allclose(np.asarray(m.sum(1)).ravel(), area, rtol=1e-10, atol=1e-8)
    assert m.data.min() > 1e-10 and m.data.max() <= 1.0
    m2 = gis.compute_indicatormatrix(x, y, rings)
    assert (m.indptr == m2.indptr).all() and (m.indices == m2.indices).all() and (m.data == m2.data).all()
    # many small batches (scratch budget of 2000 box cells) give the identical matrix
    code = ("import numpy as np, pickle, sys; sys.path.insert(0, %r); "
            "from atlite_b200 import gis, synthetic as syn; "
            "x, y = syn.make_coords(400, 300, -12.0, 33.0); "
            "m = gis.compute_indicatormatrix(x, y, syn.make_voronoi_shapes(x, y, 500)); "
            "sys.stdout.buffer.write(pickle.dumps((m.indptr, m.indices, m.data)))" % REPO)
    out = subprocess.run([sys.executable, "-c", code], check=True, capture_output=True,
                         env={**os.environ, "ATL_INDICATOR_BUDGET": "2000"}).stdout
    import pickle

    ip, ix, dat = pickle.loads(out)
    assert (ip == m.indptr).all() and (ix == m.indices).all() and (dat == m.data).all()


@pytest.mark.gpu
def test_gpu_shapes_argument_end_to_end():
    """convert_and_aggregate(shapes=...) (convert.py:235-240): the indicator matrix is
    built on the GPU and fed to the fused kernels; same result as passing it as matrix=."""
    import pandas as pd

    ds = syn.make_dataset(70, 45, 48, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0)
    c = ab.Cutout(data=ds)
    x, y = np.asarray(c.coords["x"]), np.asarray(c.coords["y"])
    rings = syn.make_voronoi_shapes(x, y, 9)
    shapes = pd.Series(rings, index=[f"region{k}" for k in range(9)])
    ind = c.indicatormatrix(shapes)
    assert sp.issparse(ind) and ind.shape == (9, 45 * 70)
    a = c.wind("Vestas_V112_3MW", shapes=shapes, aggregate_time=None)
    b = c.wind("Vestas_V112_3MW", matrix=ind, index=shapes.index, aggregate_time=None)
    assert list(a.coords[a.dims[0]]) == list(shapes.index)
    np.testing.assert_allclose(a.values, b.values, rtol=1e-5)  # float atomics: order varies run to run
    want = oracle(x, y, rings)
    np.testing.assert_allclose(ind.toarray(), want.toarray(), rtol=0, atol=2e-12)
    pu = c.pv("CSi", "latitude_optimal", shapes=shapes, per_unit=True, aggregate_time="mean")
    assert pu.shape == (9,) and (pu.values > 0).all() and (pu.values < 1).all()
