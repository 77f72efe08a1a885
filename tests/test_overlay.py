"""Overlay form of the indicator matrix (gis.py:104-145 with two polygon collections):
I[i, j] = area(dest_i ∩ orig_j) / area(orig_j).

CPU part: which form ``gis.compute_indicatormatrix`` dispatches to, argument errors raised
before any device work, the packing of holes and multipolygons for both sides, and the exact
rational checker (oracle/overlay_exact.py) against hand-computed areas and against
oracle/indicator_exact.py.  GPU part: csrc/overlay.cu against that checker on degenerate pairs and
random Voronoi sets, against the grid kernel (csrc/indicator.cu), across CRSs, and for
repeatability and empty inputs.
"""

import ctypes as C
from fractions import Fraction as Fr

import numpy as np
import pytest

import indicator_exact as IE
import overlay_exact as OX
from atlite_b200 import _lib, gis, proj, synthetic as syn


def box(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=float)


def poly(*xy):
    return np.array(xy, dtype=float)


def gj(ext, *holes):
    """GeoJSON Polygon dict, closed rings as lists."""
    close = lambda r: [list(map(float, p)) for p in r] + [list(map(float, r[0]))]  # noqa: E731
    return {"type": "Polygon", "coordinates": [close(ext)] + [close(h) for h in holes]}


def multi(*polys):
    return {"type": "MultiPolygon", "coordinates": [p["coordinates"] for p in polys]}


def exact(orig, dest):
    """{(i, j): float fraction} above the keep threshold, from the rational checker."""
    fr = OX.overlay_fractions([gis.geometry_rings(o) for o in orig], [gis.geometry_rings(d) for d in dest])
    return {k: float(v) for k, v in fr.items() if v > Fr(1, 10 ** 10)}


def assert_matches(got, want, n_dest, n_orig, atol=1e-12):
    assert got.shape == (n_dest, n_orig)
    coo = got.tocoo()
    have = {(int(i), int(j)): float(v) for i, j, v in zip(coo.row, coo.col, coo.data)}
    assert set(have) == set(want), f"pattern: extra {sorted(set(have) - set(want))}, missing {sorted(set(want) - set(have))}"
    for k, v in want.items():
        assert abs(have[k] - v) <= atol, f"{k}: {have[k]!r} vs exact {v!r}"
    for r in range(got.shape[0]):
        cols = got.indices[got.indptr[r]:got.indptr[r + 1]]
        assert (np.diff(cols) > 0).all(), "columns must ascend within a row"


# ---------------------------------------------------------------- CPU: dispatch and arguments

class _FakeLib:
    """Stands in for libatlite_b200: records which entry point is called and stops there."""

    class Called(Exception):
        pass

    def __init__(self):
        self.calls = []
        self.sides = None

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            if name == "atl_overlay_compute":  # copy the packed arrays while the caller still holds them
                self.sides = [_unpack(*args[1:6]), _unpack(*args[6:11])]
            raise _FakeLib.Called(name)
        return fn


def _read(p, ctype, n):
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(ctype)), (n,)).copy() if n else np.zeros(0, dtype=ctype)


def _unpack(n, srp, rp, holes, xy):
    srp = _read(srp, C.c_int64, n + 1)
    n_rings = int(srp[-1])
    rp = _read(rp, C.c_int64, n_rings + 1)
    return n, srp, rp, _read(holes, C.c_int8, n_rings), _read(xy, C.c_double, 2 * int(rp[-1])).reshape(-1, 2)


@pytest.fixture
def fake_lib(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    return lib


@pytest.fixture
def no_device(monkeypatch):
    def refuse():
        raise AssertionError("device work started before the arguments were checked")
    monkeypatch.setattr(_lib, "load", refuse)


def test_grid_form_for_numeric_axes(fake_lib):
    x, y = syn.make_coords(6, 4)
    import pandas as pd
    for xs in (x, list(x), pd.Index(x, name="x")):
        with pytest.raises(_FakeLib.Called):
            gis.compute_indicatormatrix(xs, y, [box(0.1, 30.1, 0.6, 30.6)], device=0)
        assert fake_lib.calls[-1][0] == "atl_indicator_compute"
    with pytest.raises(_FakeLib.Called):
        gis.compute_indicatormatrix(x=x, y=y, shapes=[box(0.1, 30.1, 0.6, 30.6)], device=0)
    assert fake_lib.calls[-1][0] == "atl_indicator_compute"


def test_overlay_form_for_collections(fake_lib):
    a, b = box(0, 0, 1, 1), box(0.5, 0.5, 2, 2)
    for orig, dest in (([a], [b]), ([gj(a)], [gj(b), None]), ([[a]], (b,)), ({"r": a}, [b]), ([a, a], [b])):
        with pytest.raises(_FakeLib.Called):
            gis.compute_indicatormatrix(orig, dest, device=0)
        assert fake_lib.calls[-1][0] == "atl_overlay_compute"
    with pytest.raises(_FakeLib.Called):
        gis.compute_indicatormatrix(orig=[a], dest=[b], orig_crs=3035, dest_crs="EPSG:3035", device=0)
    assert fake_lib.calls[-1][0] == "atl_overlay_compute"


def test_empty_first_argument(fake_lib):
    """An empty sequence is an empty orig collection, unless the third positional argument is no CRS:
    then it is an empty grid axis, which the grid form refuses with its own error."""
    sq = box(0, 0, 1, 1)
    with pytest.raises(ValueError, match="non-empty"):
        gis.compute_indicatormatrix([], [], [sq])
    with pytest.raises(ValueError, match="non-empty"):
        gis.compute_indicatormatrix(np.array([]), np.array([0.0, 1.0]), [sq], device=0)
    for args in (([], [sq]), (np.array([]), [sq], 4326, "EPSG:4326"), ([], [])):
        with pytest.raises(_FakeLib.Called):
            gis.compute_indicatormatrix(*args, device=0)
        assert fake_lib.calls[-1][0] == "atl_overlay_compute"


def test_c_entry_refuses_zero_area_orig():
    """atl_overlay_compute checks orig areas itself, before any device work."""
    lib = _lib.load()
    o = gis.pack_shapes([box(0, 0, 1, 1), None, gj(box(0, 0, 1, 1), box(0, 0, 1, 1))])
    d = gis.pack_shapes([box(0, 0, 1, 1)])
    h = C.c_void_p()
    rc = lib.atl_overlay_compute(0, 3, *map(_lib.ptr, o), 1, *map(_lib.ptr, d), C.byref(h))
    assert rc == -1 and not h.value
    assert b"orig shape 2 has zero area" in lib.atl_last_error()
    flat = gis.pack_shapes([poly((0, 0), (1, 1), (2, 2))])
    rc = lib.atl_overlay_compute(0, 1, *map(_lib.ptr, flat), 1, *map(_lib.ptr, d), C.byref(h))
    assert rc == -1 and b"orig shape 0 has zero area" in lib.atl_last_error()


def test_cutout_module_reexports_the_function():
    from atlite_b200 import cutout
    assert cutout.compute_indicatormatrix is gis.compute_indicatormatrix


@pytest.mark.parametrize("side", ["orig", "dest"])
def test_non_polygons_raise_before_device_work(no_device, side):
    good = [box(0, 0, 1, 1)]
    bad = [box(0, 0, 1, 1), {"type": "LineString", "coordinates": [[0, 0], [1, 1]]}]
    with pytest.raises(ValueError, match="Polygon"):
        gis.compute_indicatormatrix(*((bad, good) if side == "orig" else (good, bad)))


def test_zero_area_orig_raises_before_device_work(no_device):
    flat = poly((0, 0), (1, 1), (2, 2))
    with pytest.raises(ValueError, match="position 1"):
        gis.compute_indicatormatrix([box(0, 0, 1, 1), flat], [box(0, 0, 1, 1)])
    with pytest.raises(ValueError, match="position 0"):
        gis.compute_indicatormatrix([gj(box(0, 0, 1, 1), box(0, 0, 1, 1))], [box(0, 0, 1, 1)])


def test_unsupported_crs_pair_raises_before_device_work(no_device):
    with pytest.raises(NotImplementedError):
        gis.compute_indicatormatrix([box(0, 0, 1, 1)], [box(0, 0, 1, 1)], orig_crs=4326, dest_crs=32632)
    with pytest.raises(NotImplementedError):
        gis.compute_indicatormatrix([box(0, 0, 1, 1)], [box(0, 0, 1, 1)], orig_crs="EPSG:32632", dest_crs=3035)


def test_vertex_without_image_raises_before_device_work(no_device):
    with pytest.raises(ValueError, match="no image"):
        gis.compute_indicatormatrix([box(0, 0, 1e5, 1e5)], [box(0, 80, 1, 90)], orig_crs=3857, dest_crs=4326)


def test_equal_unsupported_crs_is_accepted_and_left_alone(fake_lib):
    d = box(500000.5, 5e6, 500100.25, 5.0001e6)
    with pytest.raises(_FakeLib.Called):
        gis.compute_indicatormatrix([box(5e5, 5e6, 5.001e5, 5.0001e6)], [d], orig_crs="EPSG:32632",
                                    dest_crs="EPSG:32632", device=0)
    assert np.array_equal(fake_lib.sides[1][4], d)


def test_packs_holes_and_multipolygons_on_both_sides(fake_lib):
    holed = gj(box(0, 0, 4, 4), box(1, 1, 2, 2), box(2.5, 2.5, 3, 3))
    mp = multi(gj(box(0, 0, 1, 1)), gj(box(2, 2, 5, 5), box(3, 3, 4, 4)))
    sides = ([holed, None, mp], [mp, holed])
    with pytest.raises(_FakeLib.Called):
        gis.compute_indicatormatrix(*sides, device=0)
    for (n, srp, rp, holes, xy), shapes in zip(fake_lib.sides, sides):
        assert n == len(shapes)
        want = [gis.geometry_rings(s) for s in shapes]
        assert list(np.diff(srp)) == [len(w) for w in want]
        flat = [r for w in want for r in w]
        assert list(holes) == [int(h) for _, h in flat]
        for k, (ring, _) in enumerate(flat):
            assert np.array_equal(xy[rp[k]:rp[k + 1]], ring)
    assert list(fake_lib.sides[0][1]) == [0, 3, 3, 6]  # holed (1 + 2 holes), None, mp (1 + 1 + 1 hole)


def test_host_areas_match_the_exact_checker():
    shapes = [gj(box(0, 0, 4, 4), box(1, 1, 2, 2)), multi(gj(box(0, 0, 1, 1)), gj(box(2, 2, 5, 5))),
              poly((0.1, 0.2), (3.7, 0.4), (1.3, 2.9))[::-1], None]
    got = gis._ring_shape_areas(*gis.pack_shapes(shapes))
    want = [float(OX.shape_area(gis.geometry_rings(s))) for s in shapes]
    assert np.allclose(got, want, rtol=1e-15, atol=0)


# ---------------------------------------------------------------- CPU: the exact checker

def _rings(*a):
    return [(np.asarray(r, dtype=float), h) for r, h in a]


def test_exact_checker_hand_computed():
    sq = lambda x0, y0, s: _rings((box(x0, y0, x0 + s, y0 + s), False))  # noqa: E731
    ia = OX.intersection_area
    assert ia(sq(0, 0, 2), sq(1, 1, 2)) == 1
    assert ia(sq(0, 0, 1), sq(0, 0, 1)) == 1
    assert ia(sq(0, 0, 1), sq(1, 0, 1)) == 0  # shared edge, interiors on opposite sides
    assert ia(sq(0, 0, 1), sq(1, 1, 1)) == 0  # one shared vertex
    assert ia(_rings((box(0, 0, 2, 1), False)), _rings((box(1, 0, 3, 1), False))) == 1  # collinear overlaps
    tri = _rings((poly((0, 0), (2, 0), (0, 2)), False))
    assert ia(tri, sq(0, 0, 1)) == 1 and ia(tri, sq(1, 1, 1)) == 0
    assert ia(tri, sq(0.5, 0.5, 1)) == Fr(1) - Fr(1, 2)  # the square minus the corner x + y > 2
    holed = _rings((box(0, 0, 4, 4), False), (box(1, 1, 3, 3)[::-1], True))
    assert OX.shape_area(holed) == 12
    assert ia(holed, sq(0, 0, 2)) == 3 and ia(sq(1.5, 1.5, 1), holed) == 0
    # orientation and closing vertices are free
    assert ia(_rings((box(0, 0, 2, 2)[::-1], False)), _rings((np.r_[box(1, 1, 3, 3), [[1, 1]]], False))) == 1
    # two overlapping parts of one shape count twice
    two = _rings((box(0, 0, 2, 2), False), (box(1, 0, 3, 2), False))
    assert ia(two, sq(0, 0, 3)) == 8
    # a skew quadrilateral against a triangle, by inclusion-exclusion of a known split: the triangle
    # (0,0),(4,0),(0,4) meets [1,3] x [0,1] in the trapezoid of area 2 - 1/2 (corner above x + y = 4 is empty)
    assert ia(_rings((poly((0, 0), (4, 0), (0, 4)), False)), _rings((box(1, 0, 3, 1), False))) == 2
    assert ia(_rings((poly((0, 0), (4, 0), (0, 4)), False)), _rings((box(2, 1, 4, 3), False))) == Fr(1, 2)


def test_exact_checker_agrees_with_the_cell_checker():
    x, y = syn.make_coords(7, 5, 3.0, 50.0, 0.25, 0.25)
    x1, y1 = syn.make_coords(6, 4, 10.0, 41.0, 0.1, 0.1)  # non-dyadic cell edges
    for xs, ys in ((x, y), (x1, y1)):
        regions = syn.make_voronoi_shapes(xs, ys, 4, seed=3)
        holed = [gj(box(xs[1], ys[1], xs[4], ys[3]), poly((xs[2], ys[1] + 0.01), (xs[3], ys[2]), (xs[2], ys[2])))]
        shapes = regions + holed
        want = IE.indicator_fractions(xs, ys, [gis.geometry_rings(s) for s in shapes])
        fx, fy = [Fr(float(v)) for v in xs], [Fr(float(v)) for v in ys]
        dx, dy = (fx[-1] - fx[0]) / (len(xs) - 1), (fy[-1] - fy[0]) / (len(ys) - 1)
        # the cell checker's edges are exact rationals (not always floats): the same cells here
        cells = [[([(fx[i] - dx / 2, fy[j] - dy / 2), (fx[i] + dx / 2, fy[j] - dy / 2),
                    (fx[i] + dx / 2, fy[j] + dy / 2), (fx[i] - dx / 2, fy[j] + dy / 2)], False)]
                 for j in range(len(ys)) for i in range(len(xs))]
        got = OX.overlay_fractions(cells, [gis.geometry_rings(s) for s in shapes])
        assert got == want


# ---------------------------------------------------------------- GPU

FAR_4326 = (40.0, 50.0)     # 0.25 degree cells at lon 40
FAR_3035 = (4.3e6, 3.2e6)   # EPSG:3035 metres


def _case_shapes():
    sq = box(0, 0, 1, 1)
    c = {
        "identical": ([sq], [box(0, 0, 1, 1)[::-1]]),
        "shared_edge_same_side": ([sq], [box(0, 0, 2, 1), box(0, 0, 1, 3), box(-1, -1, 1, 1)]),
        "shared_edge_opposite": ([sq], [box(1, 0, 2, 1), box(0, 1, 1, 2), box(-1, 0, 0, 1), box(0, -1, 1, 0)]),
        "collinear_partial": ([sq], [box(0.5, 0, 2, 0.5), box(0.25, 1, 0.75, 2), box(-1, 0.25, 0.5, 0.75),
                                     box(0.5, -1, 2, 0)]),
        "vertex_on_edge": ([sq], [poly((0.5, 0), (1.5, 0.5), (0.5, 1)), poly((0.5, 1), (0, 2), (1, 2)),
                                  poly((0, 0.5), (0.5, 0), (1, 0.5), (0.5, 1))]),
        "touch_vertex": ([sq], [box(1, 1, 2, 2), box(-1, -1, 0, 0), poly((1, 0.5), (2, 0), (2, 1))]),
        "nested": ([sq, box(0.25, 0.25, 0.5, 0.5)], [box(0.125, 0.125, 0.875, 0.625), box(-1, -1, 3, 3)]),
        "holes": ([gj(box(0, 0, 4, 4), box(1, 1, 3, 3))],
                  [box(1.5, 1.5, 2.5, 2.5), box(0.5, 0.5, 2, 2), box(1, 1, 3, 3), box(-1, -1, 5, 5),
                   gj(box(-1, -1, 5, 5), box(0.5, 0.5, 3.5, 3.5)), gj(box(-1, -1, 5, 5), box(0, 0, 4, 4))]),
        "multipolygons": ([multi(gj(box(0, 0, 1, 1)), gj(box(2, 0, 3, 1))), sq],
                          [multi(gj(box(0.5, 0, 2.5, 1)), gj(box(0, 2, 1, 3))), box(0, 0, 3, 1)]),
        "disjoint_boxes_overlap": ([poly((0, 0), (1, 0), (0, 1))], [poly((1, 1), (0.6, 1), (1, 0.6)),
                                                                    poly((1, 0), (1, 1), (0, 1), (0.5, 0.5))]),
    }
    # oblique edges through vertices and along each other
    c["oblique"] = ([poly((0, 0), (2, 1), (1, 3), (-1, 2))],
                    [poly((0, 0), (2, 1), (3, -1)), poly((1, 0.5), (3, 1.5), (1, 3)), poly((0.5, 1.5), (1, 3), (2, 1))])
    return c


def _shift(shapes, dx, dy, scale):
    def one(s):
        if isinstance(s, dict):
            t = s["type"]
            if t == "Polygon":
                return {"type": t, "coordinates": [[[p[0] * scale + dx, p[1] * scale + dy] for p in r]
                                                   for r in s["coordinates"]]}
            return {"type": t, "coordinates": [one({"type": "Polygon", "coordinates": p})["coordinates"]
                                               for p in s["coordinates"]]}
        return np.asarray(s) * scale + [dx, dy]
    return [one(s) for s in shapes]


CASES = _case_shapes()


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["origin", "lon40", "epsg3035"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_degenerate_pairs_exact(name, where):
    orig, dest = CASES[name]
    crs = 4326
    if where == "lon40":
        orig, dest = _shift(orig, *FAR_4326, 0.25), _shift(dest, *FAR_4326, 0.25)
    elif where == "epsg3035":
        orig, dest, crs = _shift(orig, *FAR_3035, 1000.0), _shift(dest, *FAR_3035, 1000.0), 3035
    got = gis.compute_indicatormatrix(orig, dest, crs, crs)
    assert_matches(got, exact(orig, dest), len(dest), len(orig))


@pytest.mark.gpu
def test_degenerate_pairs_expected_values():
    """The exact answers of a few cases, so the checker itself is pinned too."""
    a = gis.compute_indicatormatrix(*CASES["shared_edge_same_side"]).toarray()
    assert np.array_equal(a, [[1.0], [1.0], [1.0]])
    assert gis.compute_indicatormatrix(*CASES["shared_edge_opposite"]).nnz == 0
    assert gis.compute_indicatormatrix(*CASES["touch_vertex"]).nnz == 0
    assert gis.compute_indicatormatrix(*CASES["disjoint_boxes_overlap"]).nnz == 0  # the second only touches
    h = gis.compute_indicatormatrix(*CASES["holes"]).toarray()[:, 0] * 12
    assert np.allclose(h, [0, 1.25, 0, 12, 12 - (9 - 4), 0], rtol=0, atol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_voronoi_sets_exact(seed):
    rng = np.random.default_rng(seed)
    x, y = syn.make_coords(10, 8, 7.0 + rng.uniform(), 45.0 + rng.uniform(), 0.1, 0.1)
    orig = syn.make_voronoi_shapes(x, y, 9, seed=seed)
    dest = syn.make_voronoi_shapes(x, y, 7, seed=seed + 100, margin=0.05)
    # a holed region and a two-part region on the dest side
    dest.append(gj(box(x[1], y[1], x[7], y[6]), poly((x[2], y[2]), (x[5], y[3]), (x[3], y[5]))))
    dest.append(multi(gj(box(x[0], y[0], x[2], y[2])), gj(box(x[6], y[4], x[9], y[7]))))
    got = gis.compute_indicatormatrix(orig, dest)
    assert_matches(got, exact(orig, dest), len(dest), len(orig))
    # every dest region of the partition is covered by the orig partition: columns of the
    # partitioned rows sum to the region's share of each orig region
    tot = np.asarray(got[:7].sum(axis=0)).ravel()
    area_o = gis._ring_shape_areas(*gis.pack_shapes(orig))
    assert np.all(tot <= 1 + 1e-12) and tot @ area_o > 0


def _cell_polygons(x, y):
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    X0, Y0 = np.meshgrid(xlo, ylo)
    X1, Y1 = np.meshgrid(xhi, yhi)
    c = np.stack([X0.ravel(), Y0.ravel(), X1.ravel(), Y0.ravel(), X1.ravel(), Y1.ravel(), X0.ravel(), Y1.ravel()], 1)
    return list(c.reshape(-1, 4, 2)), (X1 - X0).ravel() * (Y1 - Y0).ravel()


@pytest.mark.gpu
def test_equals_the_grid_kernel_at_production_size():
    x, y = syn.make_coords(220, 160, -12.0 + 0.125, 33.0 + 0.125)  # Europe at 0.25 degree
    regions = syn.make_voronoi_shapes(x, y, 3000)
    cells, cell_area = _cell_polygons(x, y)
    grid = gis.compute_indicatormatrix(x, y, regions).tocsr()
    got = gis.compute_indicatormatrix(cells, regions)
    assert got.shape == grid.shape
    assert np.array_equal(got.indptr, grid.indptr) and np.array_equal(got.indices, grid.indices)
    assert np.abs(got.data - grid.data).max() <= 1e-12
    # transposed: orig = regions, dest = cells; fractions of the region instead of the cell
    region_area = gis._ring_shape_areas(*gis.pack_shapes(regions))
    want = (grid.T.tocsr().multiply(cell_area[:, None]).multiply(1.0 / region_area[None, :])).tocsr()
    want.data[want.data <= 1e-10] = 0
    want.eliminate_zeros()
    want.sort_indices()
    gotT = gis.compute_indicatormatrix(regions, cells)
    assert gotT.shape == want.shape
    assert np.array_equal(gotT.indptr, want.indptr) and np.array_equal(gotT.indices, want.indices)
    assert np.abs(gotT.data - want.data).max() <= 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("crs", [3035, "ESRI:54009", 3857])
def test_dest_crs_projects_the_vertices(crs):
    x, y = syn.make_coords(24, 16, 4.0, 46.0)
    orig = syn.make_voronoi_shapes(x, y, 20, seed=5)
    dest4326 = syn.make_voronoi_shapes(x, y, 12, seed=6, margin=0.1)
    dest = [np.stack(proj.transform(r[:, 0], r[:, 1], 4326, crs), 1) for r in dest4326]
    got = gis.compute_indicatormatrix(orig, dest, orig_crs=4326, dest_crs=crs)
    flat = np.concatenate(dest)  # projected in one call, as the package does
    flat = np.stack(proj.transform(flat[:, 0], flat[:, 1], crs, 4326), 1)
    back = np.split(flat, np.cumsum([len(r) for r in dest])[:-1])
    want = gis.compute_indicatormatrix(orig, back)
    assert got.nnz > len(dest)
    assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data, want.data)
    # and the regions keep their 4326 overlaps up to the straight-edge difference
    ref = gis.compute_indicatormatrix(orig, dest4326)
    assert abs(got - ref).max() < 1e-2


@pytest.mark.gpu
def test_bitwise_repeatable_across_calls_and_containers():
    x, y = syn.make_coords(40, 30, 5.0, 45.0)
    orig = syn.make_voronoi_shapes(x, y, 60, seed=11)
    dest = syn.make_voronoi_shapes(x, y, 45, seed=12, margin=0.3)
    as_dicts = [gj(r) for r in dest]
    a = gis.compute_indicatormatrix(orig, dest)
    b = gis.compute_indicatormatrix(orig, dest)
    c = gis.compute_indicatormatrix(orig, as_dicts)
    for m in (b, c):
        assert np.array_equal(a.indptr, m.indptr) and np.array_equal(a.indices, m.indices)
        assert a.data.tobytes() == m.data.tobytes()


@pytest.mark.gpu
def test_empty_shapes_and_collections():
    sq = box(0, 0, 1, 1)
    empty = {"type": "Polygon", "coordinates": []}
    m = gis.compute_indicatormatrix([None, sq, empty], [empty, box(0.5, 0, 1.5, 1), None])
    assert m.shape == (3, 3) and m.nnz == 1 and abs(m[1, 1] - 0.5) < 1e-15
    for orig, dest, shape in (([], [sq, sq], (2, 0)), ([sq], [], (0, 1)), ([], [], (0, 0)), ([None], [None], (1, 1)),
                              ([sq], [box(2, 2, 3, 3)], (1, 1))):
        m = gis.compute_indicatormatrix(orig, dest)
        assert m.shape == shape and m.nnz == 0
        assert m.indptr.shape == (shape[0] + 1,)


def _jitter(a, rng, ulps=4):
    """Every coordinate moved by up to ``ulps`` ulps, at random."""
    out = a.copy()
    steps = rng.integers(-ulps, ulps + 1, a.shape)
    for k in range(1, ulps + 1):
        out = np.where(steps >= k, np.nextafter(out, np.inf), out)
        out = np.where(steps <= -k, np.nextafter(out, -np.inf), out)
    return out


def _split_box(x0, y0, w, h, border):
    """The two regions left and right of ``border`` (bottom to top) in the box (x0, y0, w, h)."""
    left = np.r_[[[x0, y0]], border, [[x0, y0 + h]]]
    right = np.r_[border[:1], [[x0 + w, y0], [x0 + w, y0 + h]], border[:0:-1]]
    return left, right


@pytest.mark.gpu
@pytest.mark.parametrize("swap", [False, True])
@pytest.mark.parametrize("where", ["lon10", "lon40", "epsg3035"])
def test_borders_digitised_twice_exact(where, swap):
    """Two neighbours share a 40-vertex border; the other side's copy of it is moved by up to 4 ulps
    per coordinate.  The true overlaps across the border are slivers far below the keep threshold:
    no spurious entry, and the real entries exact to 1e-12."""
    x0, y0, w, crs = {"lon10": (10.0, 45.0, 1.0, 4326), "lon40": (40.0, 50.0, 0.25, 4326),
                      "epsg3035": (4.3e6, 3.2e6, 5e4, 3035)}[where]
    rng = np.random.default_rng(7)
    ys = y0 + w * np.linspace(0.0, 1.0, 40)
    border = np.c_[x0 + w / 2 + rng.uniform(-w / 8, w / 8, 40), ys]
    exact_pair = list(_split_box(x0, y0, w, w, border))
    moved = list(_split_box(x0, y0, w, w, _jitter(border, rng)))
    orig, dest = (exact_pair, moved) if swap else (moved, exact_pair)
    got = gis.compute_indicatormatrix(orig, dest, crs, crs)
    want = exact(orig, dest)
    assert set(want) == {(0, 0), (1, 1)}
    assert_matches(got, want, 2, 2)


@pytest.mark.gpu
def test_mixed_shape_sizes_exact():
    """Many small orig cells next to one shape covering them all and a long thin one: the candidate
    bins follow the median box, and every pair is still found."""
    x, y = syn.make_coords(20, 10, 5.0, 45.0)
    cells, _ = _cell_polygons(x, y)
    orig = cells + [box(4.0, 44.0, 11.0, 48.0), poly((4.9, 44.9), (9.9, 47.4), (9.8, 47.45))]
    dest = syn.make_voronoi_shapes(x, y, 6, seed=4) + [box(5.3, 45.3, 5.4, 45.4)]
    got = gis.compute_indicatormatrix(orig, dest)
    assert_matches(got, exact(orig, dest), len(dest), len(orig))
