"""Land eligibility: ExclusionContainer, shape_availability and Cutout.availabilitymatrix.

CPU: the projection against the EPSG worked example, cell areas, the oracle's dilation against
scipy's, the window formula, API errors.  GPU: fine masks bit for bit against the NumPy oracle of
the specification (oracle/availability_oracle.py), the reference's known answers
(test/test_gis.py:335-652, with seeded in-memory rasters in place of GeoTIFFs), availability
counts against the oracle, and the matrix end to end through Cutout.pv."""

import functools

import numpy as np
import pytest
import scipy.ndimage as ndi

import availability_oracle as AO
import atlite_b200 as ab
from atlite_b200 import gis, proj
from atlite_b200 import synthetic as syn

X0, Y0, X1, Y1 = -4.0, 56.0, 1.5, 61.0  # the reference's test cutout (test_gis.py:38-41)


def box(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=np.float64)


# ---------------------------------------------------------------- CPU
def test_laea_epsg_guidance_note_example():
    for fwd in (proj.laea_forward, AO.laea_forward):
        e, n = fwd(5.0, 50.0)  # the note gives E, N to the centimetre
        assert round(float(e), 2) == 3962799.45 and round(float(n), 2) == 2999718.85
    for inv in (proj.laea_inverse, AO.laea_inverse):
        lon, lat = inv(3962799.4509550678, 2999718.853159562)
        assert abs(lon - 5.0) < 1e-9 and abs(lat - 50.0) < 1e-9


def test_laea_round_trip_and_oracle_agree_over_europe():
    rng = np.random.default_rng(1)
    lon, lat = rng.uniform(-30, 45, 20000), rng.uniform(30, 72, 20000)
    x, y = proj.laea_forward(lon, lat)
    ox, oy = AO.laea_forward(lon, lat)
    assert np.abs(x - ox).max() < 1e-6 and np.abs(y - oy).max() < 1e-6
    x2, y2 = proj.laea_forward(*proj.laea_inverse(x, y))
    assert np.abs(x2 - x).max() <= 1e-6 and np.abs(y2 - y).max() <= 1e-6
    olon, olat = AO.laea_inverse(x, y)
    assert np.abs(olon - lon).max() < 1e-9 and np.abs(olat - lat).max() < 1e-9


def test_crs_parsing():
    assert proj.epsg(3035) == proj.epsg("EPSG:3035") == proj.epsg("epsg:3035") == 3035

    class Crs:
        def to_epsg(self):
            return 4326

    assert proj.epsg(Crs()) == 4326
    for bad in (32632, "EPSG:32632", "+proj=longlat", None):
        with pytest.raises(NotImplementedError, match="EPSG:4326 and EPSG:3035"):
            proj.epsg(bad)
    with pytest.raises(NotImplementedError):
        gis.ExclusionContainer(crs=25832)


def test_laea_cell_area_matches_fine_pixel_count():
    res = 250.0
    for lon0, lat0 in ((5.0, 50.0), (-3.0, 40.0), (20.0, 65.0)):
        lo, la = lon0 - 0.125, lat0 - 0.125
        area = proj.laea_cell_area(lo, lo + 0.25, la, la + 0.25)
        ring = np.stack(proj.laea_forward(*np.array([[lo, la], [lo + 0.25, la], [lo + 0.25, la + 0.25],
                                                     [lo, la + 0.25]]).T), axis=1)
        left, top, nx, ny = AO.window((ring[:, 0].min() - 1e3, ring[:, 1].min() - 1e3, ring[:, 0].max() + 1e3,
                                       ring[:, 1].max() + 1e3), res)
        L = (left, top, nx, ny, res)
        cnt, _ = AO.counts(np.ones((ny, nx), bool), L, 3035, (lo, 0.25, la, 0.25, 1, 1), 4326)
        perimeter = np.hypot(*np.diff(np.r_[ring, ring[:1]], axis=0).T).sum()
        assert abs(cnt[0, 0] * res * res - area) <= perimeter * res, (lon0, lat0)


@pytest.mark.parametrize("k", [1, 2, 5, 9])
def test_oracle_dilation_is_scipys(k):
    rng = np.random.default_rng(k)
    cross = ndi.generate_binary_structure(2, 1)
    for shape, p in (((37, 53), 0.02), ((5, 80), 0.05), ((64, 3), 0.1), ((40, 40), 0.0)):
        m = rng.random(shape) < p
        m[0, rng.integers(shape[1])] = True  # something on the window border
        want = ndi.binary_dilation(m, structure=cross, iterations=k, border_value=0)
        assert np.array_equal(AO.dilate(m, k), want)
        # the GPU's formulation: L1 distance to a set pixel <= k
        dist = ndi.distance_transform_cdt(~m, metric="taxicab") if m.any() else np.full(shape, k + 1)
        assert np.array_equal(dist <= k, want)


def test_padded_transform_and_shape_matches_reference_formula():
    rng = np.random.default_rng(3)
    for _ in range(200):
        res = float(rng.choice([100.0, 0.01, 250.0, 1e-3, 30.0]))
        x0, y0 = rng.uniform(-1e6, 1e6, 2) * (res / 100)
        b = (x0, y0, x0 + rng.uniform(0, 5e4) * res / 100, y0 + rng.uniform(0, 5e4) * res / 100)
        t, shape = gis.padded_transform_and_shape(b, res)
        left, bottom = ((v // res) * res for v in b[:2])
        right, top = ((v // res + 1) * res for v in b[2:])
        assert tuple(t)[:6] == (res, 0, left, 0, -res, top)
        assert shape == (int((top - bottom) / res), int((right - left) / res))


def test_api_errors_before_any_device_work():
    ex = gis.ExclusionContainer(3035, 100)
    ex.add_geometry([{"type": "LineString", "coordinates": [[4e6, 3e6], [4.1e6, 3.1e6]]}])
    with pytest.raises(ValueError, match="positive buffer"):
        ex.compute_shape_availability(box(4e6, 3e6, 4.01e6, 3.01e6), crs=3035)
    with pytest.raises(ValueError, match="differs"):
        gis.shape_availability(box(4e6, 3e6, 4.01e6, 3.01e6), gis.ExclusionContainer(3035, 100), crs=4326)
    with pytest.raises(NotImplementedError, match="availabilitymatrix"):
        gis.ExclusionContainer().compute_shape_availability(box(0, 50, 1, 51), dst_crs=4326)
    try:
        import rasterio  # noqa: F401
    except ImportError:
        ex = gis.ExclusionContainer()
        ex.add_raster("landcover.tif")
        assert ex.all_closed and not ex.all_open
        with pytest.raises(ImportError, match="rasterio"):
            ex.open_files()
    with pytest.raises(ValueError, match="north-up"):
        gis.Raster(np.zeros((3, 3)), (1, 0, 0, 0, 1, 0), 4326)
    assert "registered rasters: 0" in repr(gis.ExclusionContainer())


# ---------------------------------------------------------------- GPU helpers
def _cut(nt=2, kinds=()):
    return ab.Cutout(data=syn.make_dataset(23, 21, nt, x0=X0, y0=Y0, kinds=kinds))


def _raster(arr, transform, crs):
    return gis.Raster(arr, transform, crs), dict(array=arr, transform=transform, epsg=crs)


def _compare(shape, crs, res, rasters=(), geometries=()):
    """shape: a polygon (rings in container CRS); rasters: [(Raster, oracle raster, kwargs)];
    geometries: [(geometry, oracle kwargs, buffer, invert)]."""
    ex = gis.ExclusionContainer(crs, res)
    for r, _, kw in rasters:
        ex.add_raster(r, **kw)
    for g, _, b, inv in geometries:
        ex.add_geometry(g, buffer=b, invert=inv)
    got, t = gis.shape_availability(shape, ex)
    rings = gis.geometry_rings(shape)
    want, L, tie = AO.shape_availability(rings, proj.epsg(crs), res,
                                         [dict(raster=o, res=res, **kw) for _, o, kw in rasters],
                                         [o for _, o, _, _ in geometries])
    assert tuple(t)[:6] == (res, 0, L[0], 0, -res, L[1]) and got.shape == want.shape
    bad = (got != want) & ~tie
    assert not bad.any(), f"{bad.sum()} pixels differ (of {got.size}, {tie.sum()} excused)"
    return got, want, tie


CONCAVE = [np.array([[4.000e6, 3.000e6], [4.030e6, 3.001e6], [4.012e6, 3.012e6], [4.031e6, 3.027e6],
                     [4.001e6, 3.0305e6], [4.009e6, 3.014e6]]) + 37.5,
           np.array([[4.004e6, 3.004e6], [4.006e6, 3.008e6], [4.010e6, 3.004e6]]) + 12.25]  # exterior, hole
MULTI = {"type": "MultiPolygon", "coordinates": [
    [CONCAVE[0].tolist(), CONCAVE[1].tolist()],
    [(box(4.035e6, 3.0e6, 4.045e6, 3.02e6) + 3.3).tolist()]]}


def _landcover(seed=0, nodata_share=0.05):
    rng = np.random.default_rng(seed)
    arr = rng.integers(0, 40, (330, 480)).astype(np.uint8)
    arr[rng.random(arr.shape) < nodata_share] = 255
    return _raster(arr, (100.0, 0, 3.999e6, 0, -100.0, 3.0315e6), 3035)


# ---------------------------------------------------------------- GPU: fine masks, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [CONCAVE, MULTI], ids=["concave_hole", "multipolygon"])
@pytest.mark.parametrize("codes,invert,buffer,nodata", [
    (None, False, 0, 255), ([1, 2, 3, 7, 11], False, 100, 255), (functools.partial(np.greater_equal, 20), True, 0, 0),
    (lambda v: (v % 3) == 0, False, 750, 255), ([5, 255], True, 100, 7)])
def test_fine_mask_rasters_bit_exact(shape, codes, invert, buffer, nodata):
    r, o = _landcover()
    _compare(shape, 3035, 100, [(r, o, dict(codes=codes, invert=invert, buffer=buffer, nodata=nodata))])


@pytest.mark.gpu
def test_fine_mask_partial_and_no_overlap():
    rng = np.random.default_rng(5)
    arr = rng.integers(0, 3, (100, 120)).astype(np.int16)
    r, o = _raster(arr, (100.0, 0, 4.02e6, 0, -100.0, 3.04e6), 3035)  # covers the shape's east part only
    _compare(CONCAVE, 3035, 100, [(r, o, dict(codes=[1]))])
    far, of = _raster(arr, (100.0, 0, 5.0e6, 0, -100.0, 3.04e6), 3035)
    with pytest.raises(ValueError, match="overlap"):
        _compare(CONCAVE, 3035, 100, [(far, of, dict())])
    got, _, _ = _compare(CONCAVE, 3035, 100, [(far, of, dict(allow_no_overlap=True, nodata=0))])
    assert got.any()


@pytest.mark.gpu
def test_fine_mask_cross_crs_raster():
    """A 4326 float raster in a 3035 container: projected nearest, oracle-listed near-edge centres excused."""
    rng = np.random.default_rng(7)
    depth = rng.normal(-40, 30, (60, 90)).astype(np.float32)
    depth[3, 4] = np.nan
    lon0, lat0 = proj.laea_inverse(3.995e6, 3.035e6)
    r, o = _raster(depth, (0.01, 0, float(lon0) - 0.2, 0, -0.01, float(lat0) + 0.1), 4326)
    got, want, tie = _compare(CONCAVE, 3035, 100, [(r, o, dict(codes=lambda d: d < -50, nodata=np.nan))])
    assert (~tie).sum() > 0.99 * tie.size


@pytest.mark.gpu
@pytest.mark.parametrize("buffer,invert", [(0, False), (0, True), (260.0, False), (-180.0, False), (330.0, True)])
def test_fine_mask_geometry_exclusions(buffer, invert):
    poly = box(4.01e6, 3.005e6, 4.02e6, 3.02e6) + 0.3
    rings = [(poly, False)]
    got = _compare(CONCAVE, 3035, 100, geometries=[
        ([poly], dict(rings=rings, buffer=buffer, invert=invert), buffer, invert)])
    assert got[0].any()


@pytest.mark.gpu
def test_fine_mask_buffered_lines_and_points():
    line = np.array([[3.99e6, 3.002e6], [4.02e6, 3.025e6], [4.04e6, 3.01e6]])
    pts = np.array([[4.005e6, 3.02e6], [4.028e6, 3.004e6]])
    geoms = [{"type": "LineString", "coordinates": line.tolist()}, {"type": "MultiPoint", "coordinates": pts.tolist()}]
    _compare(MULTI, 3035, 100, geometries=[(geoms, dict(rings=[], lines=[line], points=[pts], buffer=420.0), 420.0,
                                            False)])


# ---------------------------------------------------------------- GPU: the reference's known answers
def _ref_raster(seed, values):
    t, (ny, nx) = gis.padded_transform_and_shape((X0, Y0, X1, Y1), 0.01)
    rng = np.random.default_rng(seed)
    return gis.Raster(values(rng, (ny, nx)).astype(np.int32), t, 4326)


@pytest.mark.gpu
def test_known_availability_matrix_flat():
    cut = _cut()
    shapes = [box(X0 + 1, Y0 + 1, X1 - 1, Y1 - 1)]
    I = np.asarray(cut.indicatormatrix(shapes).sum(0)).reshape(cut.shape)
    A = cut.availabilitymatrix(shapes, gis.ExclusionContainer(4326, res=0.005))
    assert A.dims == ("dim_0", "y", "x")
    assert np.allclose(I, np.asarray(A.values).sum(0))


@pytest.mark.gpu
def test_known_exclude_geometry_quarter():
    shapes = box(X0, Y0, X1, Y1)
    exclude = [box(X0 / 2 + X1 / 2, Y0 / 2 + Y1 / 2, X1, Y1)]
    area, res = (X1 - X0) * (Y1 - Y0), 0.01
    ex = gis.ExclusionContainer(4326, res=res)
    ex.add_geometry(exclude)
    m, _ = gis.shape_availability(shapes, ex)
    assert np.isclose(3 * area / 4, m.sum() * res ** 2, rtol=1e-3)
    ex = gis.ExclusionContainer(4326, res=res)
    ex.add_geometry(exclude, invert=True)
    m, _ = gis.shape_availability(shapes, ex)
    assert np.isclose(area / 4, m.sum() * res ** 2, rtol=1e-3)


@pytest.mark.gpu
def test_known_exclude_raster_ratios_and_codes():
    shapes, res = box(X0, Y0, X1, Y1), 0.01
    raster = _ref_raster(0, lambda g, s: g.random(s) < 0.25)

    def ratio(**kw):
        ex = gis.ExclusionContainer(4326, res=res)
        ex.add_raster(raster, **kw)
        m, _ = gis.shape_availability(shapes, ex)
        return m.sum() / m.size

    assert round(ratio(), 2) == 0.75 and round(ratio(invert=True), 2) == 0.25
    assert round(ratio(buffer=res), 2) < 0.75
    assert ratio(buffer=res) >= ratio(buffer=res, invert=True)
    codes = _ref_raster(1, lambda g, s: g.random(s) * 100)
    raster = codes
    assert round(ratio(codes=range(20)), 1) == 0.8
    r2 = ratio(codes=range(20), invert=True)
    assert round(r2, 1) == 0.2 and ratio(codes=lambda x: x < 20, invert=True) == r2


@pytest.mark.gpu
def test_known_partial_overlap_and_no_overlap():
    res = 0.01
    raster = _ref_raster(2, lambda g, s: g.random(s) < 0.25)
    bounds = X0 - 2, Y0, X0 + 2, Y1
    area = (bounds[2] - bounds[0]) * (bounds[3] - bounds[1])

    def avail(b, **kw):
        ex = gis.ExclusionContainer(4326, res=res)
        ex.add_raster(raster, **kw)
        m, _ = gis.shape_availability(box(*b), ex)
        return m.sum() * res ** 2

    assert np.isclose(avail(bounds, codes=[0, 1]), area / 2, rtol=1e-9)
    assert avail(bounds, nodata=0) > area / 2 > avail(bounds, nodata=1)
    far = X0 - 10.0, Y0 - 10.0, X0 - 2.0, Y0 - 2.0
    farea = (far[2] - far[0]) * (far[3] - far[1])
    with pytest.raises(ValueError):
        avail(far)
    assert avail(far, allow_no_overlap=True) == 0
    assert np.isclose(avail(far, allow_no_overlap=True, codes=[1, 255], invert=True), farea, rtol=1e-9)
    assert np.isclose(avail(far, allow_no_overlap=True, nodata=0), farea, rtol=1e-9)


@pytest.mark.gpu
def test_known_availability_matrix_rastered_and_repeatable():
    import pandas as pd

    cut = _cut()
    raster = _ref_raster(3, lambda g, s: g.random(s) < 0.25)
    shapes = pd.Series([box(X0 + 1, Y0 + 1, X1 - 1, (Y0 + Y1) / 2), box(X0 + 1, (Y0 + Y1) / 2, X1 - 1, Y1 - 1)],
                       index=pd.Index([10, 11], name="shape"))
    I = np.asarray(cut.indicatormatrix(shapes).todense())
    ex = gis.ExclusionContainer(4326, res=0.01)
    ex.add_raster(raster)
    A = cut.availabilitymatrix(shapes, ex)
    assert A.dims == ("shape", "y", "x") and list(np.asarray(A.coords["shape"])) == [10, 11]
    v = np.asarray(A.values)
    assert np.isclose(I.sum() * 0.75, v.sum(), atol=5)
    np.testing.assert_allclose(I.sum(1) * 0.75, v.sum((1, 2)), atol=5)
    np.testing.assert_array_equal(v, np.asarray(cut.availabilitymatrix(shapes, ex, nprocesses=2).values))


# ---------------------------------------------------------------- GPU: counts against the oracle
def _oracle_matrix(cut, shapes_rings, crs, res, rasters=(), geometries=(), shapes_crs=4326):
    x, y = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    grid = (x[0] - cut.dx / 2, cut.dx, y[0] - cut.dy / 2, cut.dy, len(x), len(y))
    out, ties = [], 0
    for rings in shapes_rings:
        pr = [(np.stack(proj.transform(r[:, 0], r[:, 1], shapes_crs, crs), axis=1), h) for r, h in rings]
        elig, L, _ = AO.shape_availability(pr, crs, res, rasters, geometries)
        c, t = AO.counts(elig, L, crs, grid, 4326)
        out.append(c)
        ties += t
    return np.array(out), ties


def _check_counts(A, cut, want, ties, res, crs):
    x, y = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    if crs == 4326:
        area = np.full(cut.shape, abs(cut.dx * cut.dy))
    else:
        xlo = x[0] - cut.dx / 2 + np.arange(len(x)) * cut.dx
        ylo = y[0] - cut.dy / 2 + np.arange(len(y)) * cut.dy
        area = proj.laea_cell_area(xlo[None], xlo[None] + cut.dx, ylo[:, None], ylo[:, None] + cut.dy)
    got = np.asarray(A.values)
    cnt = np.rint(got * area / (res * res)).astype(np.int64)
    np.testing.assert_allclose(got, cnt * (res * res) / area, rtol=1e-12, atol=0)
    assert np.abs(cnt - want).sum() <= 2 * ties, (np.abs(cnt - want).sum(), ties)
    if ties == 0:
        np.testing.assert_array_equal(cnt, want)


@pytest.mark.gpu
def test_counts_4326_container():
    cut = _cut()
    raster = _ref_raster(4, lambda g, s: g.integers(0, 50, s))
    xs, ys = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    rings = [gis.geometry_rings(r) for r in syn.make_voronoi_shapes(xs, ys, 4, margin=0.3)]
    ex = gis.ExclusionContainer(4326, res=0.01)
    ex.add_raster(raster, codes=[1, 2, 3, 40], buffer=0.02)
    A = cut.availabilitymatrix([[r for r, _ in g] for g in rings], ex)
    o = dict(array=np.asarray(raster.array), transform=raster.transform, epsg=4326)
    want, ties = _oracle_matrix(cut, rings, 4326, 0.01, [dict(raster=o, codes=[1, 2, 3, 40], buffer=0.02, res=0.01)])
    _check_counts(A, cut, want, ties, 0.01, 4326)


@pytest.mark.gpu
def test_counts_3035_container_overlapping_regions():
    cut = _cut()
    regions = [box(-2.5, 57.2, -0.5, 59.0), box(-1.5, 58.0, 0.8, 60.3),
               np.array([[-3.6, 56.5], [0.9, 56.9], [-1.0, 60.6]])]
    lx, ly = proj.laea_forward(-1.0, 58.5)
    coast = {"type": "LineString", "coordinates": [[lx - 8e4, ly - 5e4], [lx + 3e4, ly + 2e4], [lx + 9e4, ly - 1e4]]}
    cl = np.array(coast["coordinates"])
    r, o = _raster(np.random.default_rng(9).integers(0, 12, (900, 900)).astype(np.uint8),
                   (500.0, 0, float(lx) - 2.2e5, 0, -500.0, float(ly) + 2.2e5), 3035)
    ex = gis.ExclusionContainer(3035, res=250)
    ex.add_raster(r, codes=[0, 1, 2], buffer=300)
    ex.add_geometry([coast], buffer=2000)
    A = cut.availabilitymatrix(regions, ex, shapes_crs=4326)
    want, ties = _oracle_matrix(cut, [[(q, False)] for q in regions], 3035, 250,
                                [dict(raster=o, codes=[0, 1, 2], buffer=300, res=250)],
                                [dict(rings=[], lines=[cl], buffer=2000.0)])
    _check_counts(A, cut, want, ties, 250, 3035)


@pytest.mark.gpu
def test_counts_one_large_region():
    """One region of more than 2e7 pixels (EPSG:3035 at 100 m)."""
    cut = _cut()
    region = box(-3.8, 56.2, 1.3, 60.8)
    ex = gis.ExclusionContainer(3035, res=100)
    A = cut.availabilitymatrix([region], ex)
    pr = np.stack(proj.laea_forward(region[:, 0], region[:, 1]), axis=1)
    left, top, nx, ny = AO.window((pr[:, 0].min(), pr[:, 1].min(), pr[:, 0].max(), pr[:, 1].max()), 100)
    assert nx * ny >= 2e7
    want, ties = _oracle_matrix(cut, [[(region, False)]], 3035, 100)
    _check_counts(A, cut, want, ties, 100, 3035)


@pytest.mark.gpu
def test_matrix_end_to_end_through_pv():
    import pandas as pd
    import scipy.sparse as sp

    cut = _cut(nt=24, kinds=("pv",))
    raster = _ref_raster(6, lambda g, s: g.random(s) < 0.3)
    xs, ys = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    shapes = syn.make_voronoi_shapes(xs, ys, 5, margin=0.3)
    ex = gis.ExclusionContainer(4326, res=0.01)
    ex.add_raster(raster)
    A = np.asarray(cut.availabilitymatrix(shapes, ex).values)
    o = dict(array=np.asarray(raster.array), transform=raster.transform, epsg=4326)
    want, _ = _oracle_matrix(cut, [gis.geometry_rings(s) for s in shapes], 4326, 0.01,
                             [dict(raster=o, res=0.01)])
    Ao = want * 0.01 ** 2 / abs(cut.dx * cut.dy)
    area = np.asarray(cut.area().values)
    got = cut.pv("CSi", "latitude_optimal", matrix=sp.csr_matrix((A * area * 1.7).reshape(5, -1)),
                 index=pd.RangeIndex(5), aggregate_time=None)
    ref = cut.pv("CSi", "latitude_optimal", matrix=sp.csr_matrix((Ao * area * 1.7).reshape(5, -1)),
                 index=pd.RangeIndex(5), aggregate_time=None)
    np.testing.assert_allclose(np.asarray(got.values), np.asarray(ref.values), rtol=1e-5, atol=1e-9)
