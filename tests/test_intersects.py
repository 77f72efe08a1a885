"""General form of the intersection matrix (gis.py:148-183 with two geometry collections):
I[i, j] = 1.0 when dest_i and orig_j intersect as closed sets.

CPU part: which form ``gis.compute_intersectionmatrix`` dispatches to, the packing of every
geometry kind on both sides, argument errors raised before any device work (in Python and in the
C entry point), and the exact rational checker (oracle/intersects_exact.py) against hand-computed
cases and against oracle/intersection_exact.py's cell predicate.  GPU part: csrc/overlay.cu's
intersects test equal to that checker on degenerate and random cases, equal to the grid form
(csrc/indicator.cu) at production size, consistent with the overlay form, across CRSs, on a
polygon of 10^5 vertices, and bitwise repeatable.
"""

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import intersection_exact as IX
import intersects_exact as SX
from atlite_b200 import _lib, gis, proj, synthetic as syn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def point(x, y):
    return {"type": "Point", "coordinates": [float(x), float(y)]}


def line(*xy):
    return {"type": "LineString", "coordinates": [list(map(float, p)) for p in xy]}


def parts(shapes):
    return [gis.geometry_parts(s) for s in shapes]


def exact(orig, dest):
    return SX.intersects_matrix(parts(orig), parts(dest))


def assert_exact(got, orig, dest):
    want = exact(orig, dest)
    assert got.shape == want.shape == (len(dest), len(orig))
    assert got.has_sorted_indices and got.indices.dtype == np.int32 and got.dtype == np.float64
    assert (got.data == 1.0).all()
    a = got.toarray()
    bad = sorted({(int(i), int(j)) for i, j in zip(*np.nonzero(a != want))})
    assert not bad, f"(dest, orig) pairs that differ from the exact checker: {bad[:20]}"


def same_csr(a, b):
    return (a.shape == b.shape and np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices)
            and a.data.tobytes() == b.data.tobytes())


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
            if name == "atl_intersects_compute":  # copy the packed arrays while the caller still holds them
                self.sides = [_unpack(*args[1:6]), _unpack(*args[6:11])]
            raise _FakeLib.Called(name)
        return fn


def _read(p, ctype, n):
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(ctype)), (n,)).copy() if n else np.zeros(0, dtype=ctype)


def _unpack(n, spp, pp, kinds, xy):
    spp = _read(spp, C.c_int64, n + 1)
    n_parts = int(spp[-1])
    pp = _read(pp, C.c_int64, n_parts + 1)
    return n, spp, pp, _read(kinds, C.c_int8, n_parts), _read(xy, C.c_double, 2 * int(pp[-1])).reshape(-1, 2)


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
            gis.compute_intersectionmatrix(xs, y, [box(0.1, 30.1, 0.6, 30.6)], device=0)
        assert fake_lib.calls[-1][0] == "atl_intersection_compute"
    for kw in ({"x": x, "y": y, "shapes": [point(0.1, 30.1)]}, {"y": y, "shapes": [point(0.1, 30.1)]}):
        args = () if "x" in kw else (x,)
        with pytest.raises(_FakeLib.Called):
            gis.compute_intersectionmatrix(*args, **kw, device=0)
        assert fake_lib.calls[-1][0] == "atl_intersection_compute"


def test_general_form_for_collections(fake_lib):
    a, b = box(0, 0, 1, 1), line((0, 0), (2, 2))
    for orig, dest in (([a], [b]), ([gj(a)], [b, None]), ([[a]], (point(1, 1),)), ({"r": a}, [b]),
                       ([point(0, 0)], [a]), ([b, b], [a])):
        with pytest.raises(_FakeLib.Called):
            gis.compute_intersectionmatrix(orig, dest, device=0)
        assert fake_lib.calls[-1][0] == "atl_intersects_compute"
    with pytest.raises(_FakeLib.Called):
        gis.compute_intersectionmatrix(orig=[a], dest=[b], orig_crs=3035, dest_crs="EPSG:3035", device=0)
    assert fake_lib.calls[-1][0] == "atl_intersects_compute"


def test_empty_first_argument(fake_lib):
    """An empty sequence is an empty orig collection, unless the third positional argument is no CRS:
    then it is an empty grid axis, which the grid form refuses with its own error."""
    sq = box(0, 0, 1, 1)
    with pytest.raises(ValueError, match="non-empty"):
        gis.compute_intersectionmatrix([], [], [sq])
    with pytest.raises(ValueError, match="non-empty"):
        gis.compute_intersectionmatrix(np.array([]), np.array([0.0, 1.0]), [sq], device=0)
    for args in (([], [sq]), (np.array([]), [sq], 4326, "EPSG:4326"), ([], [])):
        with pytest.raises(_FakeLib.Called):
            gis.compute_intersectionmatrix(*args, device=0)
        assert fake_lib.calls[-1][0] == "atl_intersects_compute"


def test_packs_every_kind_on_both_sides(fake_lib):
    holed = gj(box(0, 0, 4, 4), box(1, 1, 2, 2))
    mp = multi(gj(box(0, 0, 1, 1)), gj(box(2, 2, 5, 5), box(3, 3, 4, 4)))
    mls = {"type": "MultiLineString", "coordinates": [[[0, 0], [1, 1], [2, 0]], [[5, 5], [6, 6]]]}
    mpt = {"type": "MultiPoint", "coordinates": [[0.5, 0.5], [7, 7], [8, 9]]}
    coll = {"type": "GeometryCollection", "geometries": [point(3, 3), line((0, 1), (1, 0)), gj(box(9, 9, 10, 10))]}
    ring = {"type": "LinearRing", "coordinates": [[0, 0], [1, 0], [1, 1], [0, 0]]}

    class Geo:  # anything with __geo_interface__
        __geo_interface__ = line((7, 7), (8, 8))

    sides = ([holed, None, mp, mls, point(1, 2)], [mpt, coll, ring, Geo(), box(0, 0, 1, 1)])
    with pytest.raises(_FakeLib.Called):
        gis.compute_intersectionmatrix(*sides, device=0)
    for (n, spp, pp, kinds, xy), shapes in zip(fake_lib.sides, sides):
        assert n == len(shapes)
        want = parts(shapes)
        assert list(np.diff(spp)) == [len(w) for w in want]
        flat = [p for w in want for p in w]
        assert list(kinds) == [k for k, _ in flat]
        for k, (_, c) in enumerate(flat):
            assert np.array_equal(xy[pp[k]:pp[k + 1]], c)
    assert list(fake_lib.sides[0][3]) == [0, 1, 0, 0, 1, 2, 2, 3]
    assert list(fake_lib.sides[1][3]) == [3, 3, 2, 0, 2, 2, 0]


def test_unsupported_crs_pair_raises_before_device_work(no_device):
    with pytest.raises(NotImplementedError):
        gis.compute_intersectionmatrix([box(0, 0, 1, 1)], [point(0, 0)], orig_crs=4326, dest_crs=32632)
    with pytest.raises(NotImplementedError):
        gis.compute_intersectionmatrix([line((0, 0), (1, 1))], [box(0, 0, 1, 1)], orig_crs="EPSG:32632", dest_crs=3035)


def test_vertex_without_image_raises_before_device_work(no_device):
    with pytest.raises(ValueError, match="no image"):
        gis.compute_intersectionmatrix([box(0, 0, 1e5, 1e5)], [line((0, 80), (1, 90))], orig_crs=3857, dest_crs=4326)


def test_equal_unsupported_crs_is_accepted_and_left_alone(fake_lib):
    d = np.array([[500000.5, 5e6], [500100.25, 5.0001e6]])
    with pytest.raises(_FakeLib.Called):
        gis.compute_intersectionmatrix([box(5e5, 5e6, 5.001e5, 5.0001e6)], [line(*d)], orig_crs="EPSG:32632",
                                       dest_crs="EPSG:32632", device=0)
    assert np.array_equal(fake_lib.sides[1][4], d)


def test_c_entry_checks_every_part_before_device_work():
    """atl_intersects_compute refuses malformed input on either side before it touches a device."""
    lib = _lib.load()
    good = gis.pack_geometries([box(0, 0, 1, 1), line((0, 0), (1, 1)), point(0.5, 0.5)])

    def call(o, d, n_o=None, n_d=None):
        h = C.c_void_p()
        n_o = len(o[0]) - 1 if n_o is None else n_o
        n_d = len(d[0]) - 1 if n_d is None else n_d
        rc = lib.atl_intersects_compute(0, n_o, *map(_lib.ptr, o), n_d, *map(_lib.ptr, d), C.byref(h))
        assert not h.value
        return rc, lib.atl_last_error()

    spp, pp, kinds, xy = good
    bad = {
        b"shape_part_ptr must be non-decreasing": (np.array([0, 2, 1, 3], dtype=np.int64), pp, kinds, xy),
        b"part_ptr must be non-decreasing": (spp, np.array([0, 4, 2, 7], dtype=np.int64), kinds, xy),
        b"unknown part kind": (spp, pp, np.array([0, 7, 3], dtype=np.int8), xy),
        b"non-finite vertex": (spp, pp, kinds, np.where(np.arange(len(xy))[:, None] == 5, np.nan, xy)),
    }
    for msg, b in bad.items():
        b = tuple(np.ascontiguousarray(a) for a in b)
        for o, d in ((b, good), (good, b)):
            rc, err = call(o, d)
            assert rc == -1 and msg in err, (msg, err)
    rc, err = call(good, good, n_o=-1)
    assert rc == -1 and b"negative shape count" in err
    h = C.c_void_p()
    rc = lib.atl_intersects_compute(0, 1, _lib.ptr(spp), None, None, None, 1, *map(_lib.ptr, good), C.byref(h))
    assert rc == -1 and b"NULL argument" in lib.atl_last_error()


def test_cutout_module_reexports_the_function():
    from atlite_b200 import cutout
    assert cutout.compute_intersectionmatrix is gis.compute_intersectionmatrix


def test_product_does_not_import_the_oracle():
    code = ("import sys, atlite_b200, atlite_b200.gis, atlite_b200.cutout; "
            "assert 'intersects_exact' not in sys.modules")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=REPO)


# ---------------------------------------------------------------- CPU: the exact checker

def test_exact_checker_hand_computed():
    I = lambda a, b: SX.intersects(gis.geometry_parts(a), gis.geometry_parts(b))  # noqa: E731
    sq, holed = box(0, 0, 1, 1), gj(box(0, 0, 4, 4), box(1, 1, 3, 3))
    assert I(sq, point(0.5, 0)) and I(sq, point(1, 1)) and I(sq, point(0.5, 0.5))
    assert not I(sq, point(1, 1 + 2 ** -40))
    assert not I(holed, point(2, 2)) and I(holed, point(1, 2)) and I(holed, point(0.5, 2))
    assert I(holed, box(1, 1.5, 2, 2.5)) and not I(holed, box(1.5, 1.5, 2.5, 2.5))
    assert I(holed, box(-1, -1, 5, 5)) and not I(holed, gj(box(-1, -1, 5, 5), box(-0.5, -0.5, 4.5, 4.5)))
    assert I(line((0, 0), (2, 0)), line((1, 0), (3, 0))) and I(line((0, 0), (2, 0)), line((2, 0), (3, 0)))
    assert not I(line((0, 0), (2, 0)), line((2.5, 0), (3, 0)))
    assert I(line((0, 0), (2, 0)), line((1, -1), (1, 0))) and not I(line((0, 0), (2, 0)), line((1, -1), (1, -0.5)))
    assert I(line((0, 0), (1, 1)), line((0.5, 0.5), (2, 2))) and not I(line((0, 0), (1, 1)), line((0.5, 0.6), (2, 2.1)))
    assert I(sq, box(0.25, 0.25, 0.75, 0.75)) and I(box(0.25, 0.25, 0.75, 0.75), sq)
    two = multi(gj(box(0, 0, 2, 2)), gj(box(1, 1, 3, 3)))
    assert I(two, point(1.5, 1.5))  # overlapping parts of one shape do not cancel
    flat = poly((0, 0), (1, 1), (2, 2))  # a zero-area ring: its edges only
    assert I(flat, point(1, 1)) and not I(flat, point(0.5, 0.6)) and I(flat, line((0, 1), (1, 0)))
    assert I(line((0, 0), (0, 0)), point(0, 0)) and not I(point(0, 0), point(0, 1e-300))
    assert not I(None, sq) and not I({"type": "Polygon", "coordinates": []}, sq)


@pytest.mark.parametrize("step", [0.25, 0.1, 0.3])
def test_exact_checker_agrees_with_the_cell_checker(step):
    x, y = syn.make_coords(9, 7, 3.0 + step / 2, 50.0 + step / 2, step, step)
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    rng = np.random.default_rng(int(step * 100))
    shapes = syn.make_voronoi_shapes(x, y, 5, seed=3) + syn.make_line_network(x, y, 4)[:6]
    shapes += [point(xlo[k], ylo[2]) for k in range(1, 5)] + [point(xhi[3], yhi[k]) for k in range(1, 4)]
    shapes += [point(*p) for p in np.c_[rng.uniform(x[0], x[-1], 6), rng.uniform(y[0], y[-1], 6)]]
    shapes += [gj(box(x[1], y[1], x[6], y[5]), box(x[2], y[2], x[4], y[3])), line((xlo[2], ylo[1]), (xlo[2], yhi[4]))]
    want = IX.intersectionmatrix(x, y, parts(shapes))
    assert np.array_equal(exact(_cell_polygons(x, y), shapes), want)


# ---------------------------------------------------------------- GPU

FAR_4326 = (40.0, 50.0)     # at lon 40, scaled to 0.25
FAR_3035 = (4.3e6, 3.2e6)   # EPSG:3035 metres, scaled to 1000


def _cell_polygons(x, y):
    """The reference boxes of the cells (gis.cell_edges) as polygons, in cutout.grid order."""
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    X0, Y0 = np.meshgrid(xlo, ylo)
    X1, Y1 = np.meshgrid(xhi, yhi)
    c = np.stack([X0.ravel(), Y0.ravel(), X1.ravel(), Y0.ravel(), X1.ravel(), Y1.ravel(), X0.ravel(), Y1.ravel()], 1)
    return list(c.reshape(-1, 4, 2))


def _map(c, f):
    """Nested coordinate lists with every (x, y) pair mapped by f."""
    if len(c) and np.isscalar(c[0]):
        return list(f(c))
    return [_map(v, f) for v in c]


def _shift(shapes, dx, dy, scale):
    f = lambda p: (p[0] * scale + dx, p[1] * scale + dy)  # noqa: E731

    def one(s):
        if s is None:
            return None
        if isinstance(s, dict):
            if s["type"] == "GeometryCollection":
                return {"type": s["type"], "geometries": [one(g) for g in s["geometries"]]}
            return {"type": s["type"], "coordinates": _map(s["coordinates"], f)}
        return np.asarray(s) * scale + [dx, dy]
    return [one(s) for s in shapes]


def _cases():
    sq = box(0, 0, 1, 1)
    holed = gj(box(0, 0, 4, 4), box(1, 1, 3, 3))
    return {
        "points": ([sq, holed], [point(0.5, 0), point(1, 1), point(2, 2), point(1, 2), point(3, 3), point(0.5, 0.5),
                                 point(5, 5), point(4, 2), {"type": "MultiPoint", "coordinates": [[9, 9], [2, 1]]}]),
        "lines_along_a_shared_border": ([box(0, 0, 1, 1), box(1, 0, 2, 1)],
                                        [line((1, 0), (1, 1)), line((1, -1), (1, 0.5)), line((0, 1), (2, 1)),
                                         line((1.5, 1), (3, 1)), line((2.5, 0), (3, 0)), line((0, -1), (0.5, -0.5)),
                                         line((2, 0.5), (3, 0.5))]),
        "collinear_and_t": ([line((0, 0), (2, 0)), line((0, 0), (1, 1))],
                            [line((1, 0), (3, 0)), line((2, 0), (3, 0)), line((1, -1), (1, 0)), line((2.5, 0), (3, 0)),
                             line((0.5, 0.5), (2, 2)), line((0.5, 0.6), (2, 2.1)), line((1, 2), (1, 1)),
                             line((-1, -1), (-0.5, -0.5)), line((3, 0), (2, 0), (2, -1))]),
        "polygon_in_a_hole": ([holed], [box(1.5, 1.5, 2.5, 2.5), box(1, 1.5, 2, 2.5), box(2.5, 2.5, 3, 3),
                                        box(0.25, 0.25, 0.75, 0.75), box(-1, -1, 5, 5),
                                        gj(box(-1, -1, 5, 5), box(-0.5, -0.5, 4.5, 4.5)),
                                        gj(box(-1, -1, 5, 5), box(0, 0, 4, 4)), poly((2, 1), (3, 2), (2, 3), (1, 2))]),
        "nested": ([sq, box(0.25, 0.25, 0.5, 0.5)], [box(0.125, 0.125, 0.875, 0.625), box(-1, -1, 3, 3),
                                                      box(0.3, 0.3, 0.4, 0.4)]),
        "multi_part": ([multi(gj(box(0, 0, 1, 1)), gj(box(2, 0, 3, 1))),
                        {"type": "MultiLineString", "coordinates": [[[0, 2], [3, 2]], [[5, 5], [6, 6]]]},
                        {"type": "MultiPoint", "coordinates": [[0.5, 0.5], [10, 10]]}],
                       [box(2.25, 0.25, 2.5, 0.5), point(5.5, 5.5), multi(gj(box(9, 9, 11, 11)), gj(box(-1, 1.5, 0, 3))),
                        {"type": "GeometryCollection", "geometries": [point(1.5, 0.5), line((1.5, 3), (1.5, 2.5))]},
                        line((1.5, 1.5), (1.5, 2.5)), point(1.5, 0.5)]),
        "identical": ([sq, holed, line((0, 0), (1, 1)), point(0.25, 0.75)],
                      [box(0, 0, 1, 1)[::-1], gj(box(0, 0, 4, 4), box(1, 1, 3, 3)), line((1, 1), (0, 0)),
                       point(0.25, 0.75)]),
        "overlapping_parts": ([multi(gj(box(0, 0, 2, 2)), gj(box(1, 1, 3, 3)))],
                              [point(1.5, 1.5), box(1.25, 1.25, 1.75, 1.75), point(0.5, 2.5)]),
        "zero_area_rings": ([poly((0, 0), (1, 1), (2, 2)), poly((0, 3), (1, 3)), poly((5, 5))],
                            [point(1, 1), point(0.5, 0.6), line((0, 1), (1, 0)), box(0.4, 0.4, 0.6, 0.6),
                             point(0.5, 3), point(5, 5), box(4, 4, 6, 6), line((0, 2.5), (0.5, 2.5))]),
        "empty": ([None, sq, {"type": "Polygon", "coordinates": []}, {"type": "MultiPoint", "coordinates": []}],
                  [{"type": "LineString", "coordinates": []}, point(0.5, 0.5), None, sq]),
    }


CASES = _cases()


@pytest.mark.gpu
@pytest.mark.parametrize("swap", [False, True])
@pytest.mark.parametrize("where", ["origin", "lon40", "epsg3035"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_degenerate_cases_exact(name, where, swap):
    orig, dest = CASES[name]
    crs = 4326
    if where == "lon40":
        orig, dest = _shift(orig, *FAR_4326, 0.25), _shift(dest, *FAR_4326, 0.25)
    elif where == "epsg3035":
        orig, dest, crs = _shift(orig, *FAR_3035, 1000.0), _shift(dest, *FAR_3035, 1000.0), 3035
    if swap:
        orig, dest = dest, orig
    got = gis.compute_intersectionmatrix(orig, dest, crs, crs)
    assert_exact(got, orig, dest)


@pytest.mark.gpu
def test_degenerate_cases_expected_values():
    """The answers of a few cases, so the checker itself is pinned too."""
    a = gis.compute_intersectionmatrix(*CASES["points"]).toarray()
    assert np.array_equal(a[:, 1], [1, 1, 0, 1, 1, 1, 0, 1, 1]) and np.array_equal(a[:, 0], [1, 1, 0, 0, 0, 1, 0, 0, 0])
    b = gis.compute_intersectionmatrix(*CASES["polygon_in_a_hole"]).toarray()[:, 0]
    assert np.array_equal(b, [0, 1, 1, 1, 1, 0, 1, 1])
    c = gis.compute_intersectionmatrix(*CASES["collinear_and_t"]).toarray()
    assert np.array_equal(c[:, 0], [1, 1, 1, 0, 0, 0, 0, 0, 1]) and np.array_equal(c[:, 1], [0, 0, 0, 0, 1, 0, 1, 0, 0])


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_random_sets_exact(seed):
    rng = np.random.default_rng(seed)
    x, y = syn.make_coords(12, 9, 7.0 + rng.uniform(), 45.0 + rng.uniform(), 0.1, 0.1)
    pts = np.c_[rng.uniform(x[0] - 0.1, x[-1] + 0.1, 40), rng.uniform(y[0] - 0.1, y[-1] + 0.1, 40)]
    regions = syn.make_voronoi_shapes(x, y, 9, seed=seed)
    lines = syn.make_line_network(x, y, 8, seed=seed + 50)
    orig = regions + lines[:10] + [point(*p) for p in pts[:20]] + [point(*regions[0][1]), point(*regions[2][0])]
    dest = (syn.make_voronoi_shapes(x, y, 7, seed=seed + 100, margin=0.05) + lines[5:15] +
            [point(*p) for p in pts[15:]] + [{"type": "MultiPoint", "coordinates": pts[:3].tolist()}])
    dest.append(gj(box(x[1], y[1], x[7], y[6]), poly((x[2], y[2]), (x[5], y[3]), (x[3], y[5]))))
    dest.append(line(regions[1][0], regions[1][1], regions[1][2]))  # along region 1's border
    got = gis.compute_intersectionmatrix(orig, dest)
    assert_exact(got, orig, dest)
    assert got.nnz > len(dest)


@pytest.mark.gpu
@pytest.mark.parametrize("step", [0.25, 0.1, 0.3])
def test_equals_the_grid_form_at_production_size(step):
    """orig = the reference boxes of the 220 x 160 cells as polygons: identical to the grid form, and
    the exact transpose with the sides swapped."""
    x, y = syn.make_coords(220, 160, -12.0 + step / 2, 33.0 + step / 2, step, step)
    rng = np.random.default_rng(int(step * 100))
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    pts = [point(*p) for p in np.c_[rng.uniform(x[0], x[-1], 3000), rng.uniform(y[0], y[-1], 3000)]]
    pts += [point(xlo[i], ylo[j]) for i, j in zip(rng.integers(1, 220, 500), rng.integers(1, 160, 500))]
    pts += [point(xhi[i], y[j]) for i, j in zip(rng.integers(0, 219, 500), rng.integers(0, 160, 500))]
    dest = syn.make_voronoi_shapes(x, y, 3000) + syn.make_line_network(x, y, 1000) + pts
    cells = _cell_polygons(x, y)
    grid = gis.compute_intersectionmatrix(x, y, dest).tocsr()
    got = gis.compute_intersectionmatrix(cells, dest)
    assert got.shape == grid.shape
    assert np.array_equal(got.indptr, grid.indptr) and np.array_equal(got.indices, grid.indices)
    assert np.array_equal(got.data, grid.data)
    want = grid.T.tocsr()
    want.sort_indices()
    gotT = gis.compute_intersectionmatrix(dest, cells)
    assert gotT.shape == want.shape
    assert np.array_equal(gotT.indptr, want.indptr) and np.array_equal(gotT.indices, want.indices)
    assert np.array_equal(gotT.data, want.data)


@pytest.mark.gpu
def test_every_overlay_entry_is_an_intersection():
    x, y = syn.make_coords(40, 30, 5.0, 45.0)
    orig = syn.make_voronoi_shapes(x, y, 60, seed=11)
    dest = syn.make_voronoi_shapes(x, y, 45, seed=12, margin=0.3)
    area = gis.compute_indicatormatrix(orig, dest)
    got = gis.compute_intersectionmatrix(orig, dest)
    assert area.nnz > 0 and (area != 0).multiply(got).nnz == area.nnz
    for s in (orig, dest):  # a partition: every region meets itself and its neighbours
        m = gis.compute_intersectionmatrix(s, s)
        assert (m.diagonal() == 1).all() and (m != m.T).nnz == 0
        assert m.nnz > gis.compute_indicatormatrix(s, s).nnz  # neighbours only touch


@pytest.mark.gpu
@pytest.mark.parametrize("crs", [3035, "ESRI:54009", 3857])
def test_dest_crs_projects_the_vertices(crs):
    x, y = syn.make_coords(24, 16, 4.0, 46.0)
    orig = syn.make_voronoi_shapes(x, y, 20, seed=5) + syn.make_line_network(x, y, 6, seed=9)
    dest4326 = syn.make_voronoi_shapes(x, y, 12, seed=6, margin=0.1)
    lines4326 = [np.asarray(s["coordinates"]) for s in syn.make_line_network(x, y, 8, seed=7)]
    dest = [np.stack(proj.transform(r[:, 0], r[:, 1], 4326, crs), 1) for r in dest4326]
    dest += [line(*np.stack(proj.transform(r[:, 0], r[:, 1], 4326, crs), 1)) for r in lines4326]
    got = gis.compute_intersectionmatrix(orig, dest, orig_crs=4326, dest_crs=crs)
    flat = np.concatenate([gis.geometry_parts(d)[0][1] for d in dest])  # projected in one call, as the package does
    flat = np.stack(proj.transform(flat[:, 0], flat[:, 1], crs, 4326), 1)
    back = np.split(flat, np.cumsum([len(gis.geometry_parts(d)[0][1]) for d in dest])[:-1])
    back = back[:len(dest4326)] + [line(*b) for b in back[len(dest4326):]]
    want = gis.compute_intersectionmatrix(orig, back)
    assert got.nnz > len(dest)
    assert same_csr(got, want)
    assert_exact(want, orig, back)


@pytest.mark.gpu
def test_long_polygon_against_short_lines():
    """One polygon of 10^5 vertices: the band index finds the few edges each short line can meet."""
    n = 100_000
    t = np.linspace(0.0, 2 * np.pi, n, endpoint=False)
    r = 3.0 + 0.4 * np.sin(37 * t) + 0.1 * np.sin(401 * t)
    big = np.c_[10.0 + r * np.cos(t), 50.0 + r * np.sin(t)]
    rng = np.random.default_rng(3)
    a = np.c_[rng.uniform(6.3, 13.7, 1500), rng.uniform(46.3, 53.7, 1500)]
    lines = [line(p, p + rng.uniform(-0.05, 0.05, 2), p + rng.uniform(-0.05, 0.05, 2)) for p in a]
    lines += [line(big[k], big[k + 1]) for k in range(0, n, 20_000)]  # along one of its edges
    lines += [point(*big[k]) for k in range(7, n, 25_000)]  # its vertices
    got = gis.compute_intersectionmatrix([big], lines)
    shape = SX.Shape(gis.geometry_parts(big))
    want = np.array([SX.shapes_intersect(SX.Shape(gis.geometry_parts(s)), shape) for s in lines], dtype=float)
    assert np.array_equal(got.toarray()[:, 0], want)
    assert 0 < want.sum() < len(lines)
    gotT = gis.compute_intersectionmatrix(lines, [big])
    assert np.array_equal(gotT.toarray()[0], want)


@pytest.mark.gpu
def test_bitwise_repeatable_across_calls_and_containers():
    x, y = syn.make_coords(40, 30, 5.0, 45.0)
    orig = syn.make_voronoi_shapes(x, y, 60, seed=11) + syn.make_line_network(x, y, 30, seed=2)
    dest = syn.make_voronoi_shapes(x, y, 45, seed=12, margin=0.3)
    pts = np.c_[np.linspace(x[0], x[-1], 500), np.linspace(y[0], y[-1], 500)]
    a = gis.compute_intersectionmatrix(orig, dest + [point(*p) for p in pts])
    b = gis.compute_intersectionmatrix(orig, dest + [point(*p) for p in pts])
    c = gis.compute_intersectionmatrix(orig, [gj(r) for r in dest] + [point(*p) for p in pts])
    assert same_csr(a, b) and same_csr(a, c)


@pytest.mark.gpu
def test_empty_shapes_and_collections():
    sq = box(0, 0, 1, 1)
    empty = {"type": "Polygon", "coordinates": []}
    m = gis.compute_intersectionmatrix([None, sq, empty], [empty, line((1, 1), (2, 2)), None])
    assert m.shape == (3, 3) and m.nnz == 1 and m[1, 1] == 1.0
    for orig, dest, shape in (([], [sq, sq], (2, 0)), ([sq], [], (0, 1)), ([], [], (0, 0)), ([None], [None], (1, 1)),
                              ([sq], [box(2, 2, 3, 3)], (1, 1)), ([point(0, 0)], [point(0, 1)], (1, 1))):
        m = gis.compute_intersectionmatrix(orig, dest)
        assert m.shape == shape and m.nnz == 0
        assert m.indptr.shape == (shape[0] + 1,)
