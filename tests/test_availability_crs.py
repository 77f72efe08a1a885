"""Availability in World Mollweide (ESRI:54009) and Web Mercator (EPSG:3857), and windows in row bands.

CPU: atlite_b200.proj against independent restatements of both projections (below: Mercator by the
Gudermannian, Mollweide by bisection in extended precision), round trips, the Mollweide Newton
iteration against mpmath, the cell areas against a fine-pixel count, CRS parsing, and pyproj where
it is installed.  GPU: fine masks against the NumPy oracle (oracle/availability_oracle.py, which
projects with atlite_b200.proj), availability counts for both containers, and banded windows equal
to the one-pass result bit for bit."""

import numpy as np
import pytest

import availability_oracle as AO
import atlite_b200 as ab
from atlite_b200 import availability, gis, proj
from atlite_b200 import synthetic as syn

R = 6378137.0
MOLL = "ESRI:54009"


# ---------------------------------------------------------------- restatements
def merc_forward(lon, lat):
    lon, lat = np.asarray(lon, float), np.asarray(lat, float)
    return R * np.pi * lon / 180.0, R * np.log(np.tan(np.pi / 4 + np.radians(lat) / 2))


def merc_inverse(x, y):
    return np.degrees(np.asarray(x, float) / R), np.degrees(2 * np.arctan(np.exp(np.asarray(y, float) / R)) - np.pi / 2)


def moll_forward(lon, lat):
    """delta = pi / 2 - |theta| by 200 bisection steps on 2 delta - sin 2 delta = pi (1 - sin |phi|)
    = 2 pi sin^2((pi / 2 - |phi|) / 2) (2 theta + sin 2 theta = pi sin phi, with theta and phi near
    the pole as the small differences), in long double."""
    ld = np.longdouble
    pi = ld("3.14159265358979323846264338327950288")
    phi = np.asarray(lat, ld) * pi / 180
    rhs = 2 * pi * np.sin((pi / 2 - np.abs(phi)) / 2) ** 2
    lo, hi = np.zeros(phi.shape, ld), np.full(phi.shape, pi / 2)
    for _ in range(200):
        mid = (lo + hi) / 2
        below = 2 * mid - np.sin(2 * mid) < rhs
        lo, hi = np.where(below, mid, lo), np.where(below, hi, mid)
    d = (lo + hi) / 2
    lam = np.asarray(lon, ld) * pi / 180
    return (np.float64(2 * np.sqrt(ld(2)) / pi * R * lam * np.sin(d)),
            np.float64(np.sign(phi) * np.sqrt(ld(2)) * R * np.cos(d)))


def moll_inverse(x, y):
    ld = np.longdouble
    pi = ld("3.14159265358979323846264338327950288")
    th = np.arcsin(np.asarray(y, ld) / (np.sqrt(ld(2)) * R))
    phi = np.arcsin((2 * th + np.sin(2 * th)) / pi)
    lam = pi * np.asarray(x, ld) / (2 * np.sqrt(ld(2)) * R * np.cos(th))
    return np.float64(lam * 180 / pi), np.float64(phi * 180 / pi)


def _globe(lat_max, n=40000, seed=0):
    rng = np.random.default_rng(seed)
    lon = np.r_[rng.uniform(-180, 180, n), -180.0, 180.0, 0.0, 180.0, -180.0]
    lat = np.r_[rng.uniform(-lat_max, lat_max, n), 0.0, 0.0, lat_max, -lat_max, lat_max]
    return lon, lat


# ---------------------------------------------------------------- CPU
@pytest.mark.parametrize("crs,fwd,inv,lat_max", [(3857, merc_forward, merc_inverse, 85.05),
                                                  (MOLL, moll_forward, moll_inverse, 89.999)])
def test_projection_matches_restatement_over_the_globe(crs, fwd, inv, lat_max):
    lon, lat = _globe(lat_max)
    x, y = proj.transform(lon, lat, 4326, crs)
    ox, oy = fwd(lon, lat)
    assert np.abs(x - ox).max() <= 1e-6 and np.abs(y - oy).max() <= 1e-6
    glon, glat = proj.transform(x, y, crs, 4326)
    olon, olat = inv(x, y)
    assert np.abs(glat - olat).max() <= 1e-9
    # near the poles a metre spans many degrees of longitude, and the float coordinates of a point
    # fix its longitude only to ~1e-10 of itself: compare longitudes on the ground
    assert (np.abs(glon - olon) * np.cos(np.radians(lat))).max() <= 1e-9


@pytest.mark.parametrize("crs,lat_max", [(3857, 85.05), (MOLL, 89.999), (3035, 89.0)])
def test_round_trips(crs, lat_max):
    lon, lat = _globe(lat_max, seed=1)
    if crs == 3035:
        lon, lat = lon / 2, np.abs(lat)  # LAEA Europe: the hemisphere around its centre
    x, y = proj.transform(lon, lat, 4326, crs)
    glon, glat = proj.transform(x, y, crs, 4326)
    assert np.abs(glat - lat).max() <= 1e-9
    assert (np.abs(glon - lon) * np.cos(np.radians(lat))).max() <= 1e-9
    x2, y2 = proj.transform(glon, glat, 4326, crs)
    assert np.abs(x2 - x).max() <= 1e-6 and np.abs(y2 - y).max() <= 1e-6
    # every pair goes through lon / lat
    for other in (3857, MOLL, 3035):
        if other != crs:
            u, v = proj.transform(x, y, crs, other)
            want = proj.transform(glon, glat, 4326, other)
            ok = np.isfinite(want[0])
            assert np.array_equal(u[ok], want[0][ok]) and np.array_equal(v[ok], want[1][ok])


def test_mollweide_newton_converges_against_mpmath():
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 30
    lats = np.r_[-90.0, 90.0, 0.0, 1e-300, -1e-12, 45.0, -60.0, np.linspace(-89.9, 89.9, 37),
                 90 - np.logspace(-13, 0, 27), -(90 - np.logspace(-10, 0, 11))]
    phis = np.radians(lats)
    got = proj.mollweide_delta(phis)
    for phi, d in zip(phis, got):
        if abs(phi) >= np.pi / 2:
            continue  # float(pi / 2) is the pole itself: checked below
        rhs = 2 * mp.pi * mp.sin((mp.pi / 2 - abs(mp.mpf(float(phi)))) / 2) ** 2  # pi (1 - sin |phi|)
        lo, hi = mp.mpf(0), mp.pi / 2
        for _ in range(110):
            mid = (lo + hi) / 2
            lo, hi = (mid, hi) if 2 * mid - mp.sin(2 * mid) < rhs else (lo, mid)
        want = (lo + hi) / 2
        assert abs(float(d) - float(want)) <= 1e-15, (phi, d, want)
    assert got[0] == 0.0 and got[1] == 0.0  # theta = -pi/2, pi/2 exactly at the poles
    x, y = proj.mollweide_forward([0.0, 123.0], [90.0, -90.0])
    assert x[0] == 0.0 and y[0] == np.sqrt(2) * R and y[1] == -np.sqrt(2) * R


@pytest.mark.parametrize("crs,area_fn,cells", [
    (MOLL, proj.mollweide_cell_area, ((5.0, 50.0), (-170.0, 75.0), (179.75, -40.0), (0.0, 0.0))),
    (3857, proj.mercator_cell_area, ((5.0, 50.0), (-170.0, 75.0), (179.75, -40.0), (0.0, 0.0)))])
def test_cell_area_matches_fine_pixel_count(crs, area_fn, cells):
    for lon0, lat0 in cells:
        lo, la = lon0 - 0.125, lat0 - 0.125
        area = area_fn(lo, lo + 0.25, la, la + 0.25)
        assert area == proj.cell_area(crs, lo, lo + 0.25, la, la + 0.25)
        t = np.linspace(0, 1, 64)
        outline = np.r_[np.c_[lo + 0.25 * t, np.full_like(t, la)], np.c_[np.full_like(t, lo + 0.25), la + 0.25 * t],
                        np.c_[lo + 0.25 * t[::-1], np.full_like(t, la + 0.25)], np.c_[np.full_like(t, lo), la + 0.25 * t[::-1]]]
        ring = np.stack(proj.transform(outline[:, 0], outline[:, 1], 4326, crs), axis=1)
        res = float(np.sqrt(area) / 120)
        left, top, nx, ny = AO.window((ring[:, 0].min() - 3 * res, ring[:, 1].min() - 3 * res,
                                       ring[:, 0].max() + 3 * res, ring[:, 1].max() + 3 * res), res)
        cnt, _ = AO.counts(np.ones((ny, nx), bool), (left, top, nx, ny, res), proj.epsg(crs),
                           (lo, 0.25, la, 0.25, 1, 1), 4326)
        perimeter = np.hypot(*np.diff(ring, axis=0).T).sum()
        assert abs(cnt[0, 0] * res * res - area) <= perimeter * res, (lon0, lat0)


def test_crs_parsing():
    assert proj.epsg(3857) == proj.epsg("EPSG:3857") == proj.epsg("epsg:3857") == 3857
    assert proj.epsg("ESRI:54009") == proj.epsg(" esri:54009") == proj.epsg(MOLL) == MOLL

    class Pyproj:  # pyproj's CRS("ESRI:54009"): no EPSG code, an ESRI authority
        def to_epsg(self):
            return None

        def to_authority(self):
            return ("ESRI", "54009")

    class Other(Pyproj):
        def to_authority(self):
            return ("ESRI", "54030")

    assert proj.epsg(Pyproj()) == MOLL
    assert proj.name(Pyproj()) == "ESRI:54009" and proj.name(3857) == "EPSG:3857"
    for bad in (54009, "EPSG:54009", "ESRI:54030", Other()):
        with pytest.raises(NotImplementedError, match="EPSG:4326 and EPSG:3035"):
            proj.epsg(bad)
    assert repr(gis.Raster(np.zeros((2, 2)), (1.0, 0, 0, 0, -1.0, 0), MOLL)) == "<Raster 2 x 2 ESRI:54009>"
    gis.ExclusionContainer(crs="ESRI:54009", res=100)
    gis.ExclusionContainer(crs=3857, res=100)


def test_points_without_an_image():
    x, y = proj.transform([0.0, 10.0], [90.0, -90.0], 4326, 3857)
    assert np.isnan(x).all() and np.isnan(y).all()
    lon, lat = proj.transform([0.0, 1.9e7, 1.7e7], [9.1e6, 0.0, 5e6], MOLL, 4326)
    assert np.isnan(lon).all() and np.isnan(lat).all()
    assert np.isnan(proj.transform([2.1e7], [0.0], 3857, 4326)[0]).all()
    with pytest.raises(ValueError, match="EPSG:3857"):
        availability._parts([np.array([[0.0, 80.0], [10.0, 90.0], [10.0, 80.0]])], 4326, 3857, polygonal=True)


def test_against_pyproj():
    pyproj = pytest.importorskip("pyproj")
    for crs, lat_max in (("EPSG:3857", 85.05), ("ESRI:54009", 89.9)):
        lon, lat = _globe(lat_max, n=5000, seed=2)
        t = pyproj.Transformer.from_crs("EPSG:4326", crs, always_xy=True)
        px, py = t.transform(lon, lat)
        x, y = proj.transform(lon, lat, 4326, crs)
        assert np.abs(x - px).max() <= 1e-3 and np.abs(y - py).max() <= 1e-3
        assert proj.epsg(pyproj.CRS(crs)) == proj.epsg(crs)


# ---------------------------------------------------------------- GPU helpers
def box(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=np.float64)


def _outline(x0, y0, x1, y1, n=16):
    """A lon / lat box with n points per side, so that its projection keeps its shape."""
    t = np.linspace(0, 1, n, endpoint=False)
    return np.r_[np.c_[x0 + (x1 - x0) * t, np.full_like(t, y0)], np.c_[np.full_like(t, x1), y0 + (y1 - y0) * t],
                 np.c_[x1 - (x1 - x0) * t, np.full_like(t, y1)], np.c_[np.full_like(t, x0), y1 - (y1 - y0) * t]]


class InCrs(list):
    """A geometry collection with a ``.crs``."""

    def __init__(self, geoms, crs):
        super().__init__(geoms)
        self.crs = crs


def _in(crs, ring, src=4326):
    return np.stack(proj.transform(ring[:, 0], ring[:, 1], src, crs), axis=1)


def _compare(shape, crs, res, rasters=(), geometries=()):
    """As test_availability._compare: rasters [(Raster, kwargs)], geometries [(geometry, oracle
    kwargs, buffer, invert)]; the shape's rings are in the container CRS."""
    ex = gis.ExclusionContainer(crs, res)
    for r, kw in rasters:
        ex.add_raster(r, **kw)
    for g, _, b, inv in geometries:
        ex.add_geometry(g, buffer=b, invert=inv)
    got, t = gis.shape_availability(shape, ex)
    orasters = [dict(raster=dict(array=np.asarray(r.array), transform=r.transform, epsg=r.epsg), res=res, **kw)
                for r, kw in rasters]
    want, L, tie = AO.shape_availability(gis.geometry_rings(shape), proj.epsg(crs), res, orasters,
                                         [o for _, o, _, _ in geometries])
    assert tuple(t)[:6] == (res, 0, L[0], 0, -res, L[1]) and got.shape == want.shape
    bad = (got != want) & ~tie
    assert not bad.any(), f"{bad.sum()} pixels differ (of {got.size}, {tie.sum()} excused)"
    assert (~tie).sum() > 0.98 * tie.size
    return got


# ---------------------------------------------------------------- GPU: fine masks
@pytest.mark.gpu
def test_fine_mask_mollweide_with_4326_and_3035_rasters():
    rng = np.random.default_rng(3)
    shape = _in(MOLL, _outline(8.0, 47.0, 8.6, 47.4))
    depth = rng.normal(-40, 30, (60, 100)).astype(np.float32)
    depth[5, 7] = np.nan
    sea = gis.Raster(depth, (0.01, 0, 7.95, 0, -0.01, 47.45), 4326)
    lx, ly = proj.laea_forward(8.3, 47.2)
    lc = gis.Raster(rng.integers(0, 20, (700, 700)).astype(np.uint8), (100.0, 0, float(lx) - 3.5e4, 0, -100.0,
                                                                        float(ly) + 3.5e4), 3035)
    got = _compare([shape], MOLL, 100, [(sea, dict(codes=lambda d: d < -50, nodata=np.nan)),
                                        (lc, dict(codes=[1, 2, 3], buffer=150))])
    assert got.any() and not got.all()


@pytest.mark.gpu
def test_fine_mask_mercator_with_mollweide_raster():
    rng = np.random.default_rng(4)
    shape = _in(3857, _outline(-70.0, 60.0, -69.5, 60.3))
    mx, my = proj.mollweide_forward(-69.75, 60.15)
    r = gis.Raster(rng.integers(0, 5, (500, 400)).astype(np.int16), (100.0, 0, float(mx) - 2e4, 0, -100.0,
                                                                      float(my) + 2.5e4), MOLL)
    got = _compare([shape], 3857, 200, [(r, dict(codes=[0], nodata=0))])
    assert got.any() and not got.all()


@pytest.mark.gpu
@pytest.mark.parametrize("crs", [MOLL, 3857])
def test_fine_mask_buffered_geometry_given_in_4326(crs):
    shape = _in(crs, _outline(20.0, 65.0, 20.8, 65.4))
    line = np.array([[19.9, 65.1], [20.4, 65.35], [20.9, 65.05]])
    poly = _outline(20.5, 65.15, 20.7, 65.3, 4)
    geoms = InCrs([{"type": "LineString", "coordinates": line.tolist()},
                   {"type": "Polygon", "coordinates": [poly.tolist()]}], 4326)
    o = dict(rings=[(_in(crs, poly), False)], lines=[_in(crs, line)], buffer=900.0)
    got = _compare([shape], crs, 150, geometries=[(geoms, o, 900.0, False)])
    assert got.any() and not got.all()


# ---------------------------------------------------------------- GPU: availability matrices
def _matrix_case(crs, res):
    """A 4326 cutout at the antimeridian above 70 N, shapes given in 4326 and one given in the
    container CRS that reaches outside the Mollweide ellipse; a 4326 raster and a buffered line."""
    cut = ab.Cutout(data=syn.make_dataset(24, 20, 2, x0=174.125, y0=68.125, kinds=()))
    shapes = [_outline(174.5, 69.0, 180.0, 71.5), _outline(176.0, 71.0, 179.5, 72.5)]
    t, shp = gis.padded_transform_and_shape((174.0, 68.0, 180.0, 73.0), 0.02)
    lc = np.random.default_rng(5).integers(0, 8, shp).astype(np.uint8)
    raster = gis.Raster(lc, t, 4326)
    ex = gis.ExclusionContainer(crs, res=res)
    ex.add_raster(raster, codes=[1, 2], nodata=1)
    line = np.array([[175.0, 70.0], [178.0, 71.2], [179.9, 70.4]])
    ex.add_geometry(InCrs([{"type": "LineString", "coordinates": line.tolist()}], 4326), buffer=3000)
    o = dict(raster=dict(array=lc, transform=tuple(t)[:6], epsg=4326), codes=[1, 2], nodata=1, res=res)
    og = dict(rings=[], lines=[_in(crs, line)], buffer=3000.0)
    return cut, shapes, ex, o, og


def _oracle_counts(cut, rings_in_crs, crs, res, rasters, geometries):
    x, y = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    grid = (x[0] - cut.dx / 2, cut.dx, y[0] - cut.dy / 2, cut.dy, len(x), len(y))
    out, ties = [], 0
    for ring in rings_in_crs:
        elig, L, _ = AO.shape_availability([(ring, False)], proj.epsg(crs), res, rasters, geometries)
        c, t = AO.counts(elig, L, proj.epsg(crs), grid, 4326)
        out.append(c)
        ties += t
    return np.array(out), ties


@pytest.mark.gpu
@pytest.mark.parametrize("crs,res", [(MOLL, 1000.0), (3857, 2500.0)])
def test_counts_at_the_antimeridian_above_70n(crs, res):
    cut, shapes, ex, o, og = _matrix_case(crs, res)
    rings = [_in(crs, s) for s in shapes]
    A = cut.availabilitymatrix(shapes, ex)
    want, ties = _oracle_counts(cut, rings, crs, res, [o], [og])
    x, y = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    xlo, ylo = x - cut.dx / 2, y - cut.dy / 2
    area = proj.cell_area(crs, xlo[None], xlo[None] + cut.dx, ylo[:, None], ylo[:, None] + cut.dy)
    got = np.asarray(A.values)
    cnt = np.rint(got * area / (res * res)).astype(np.int64)
    np.testing.assert_allclose(got, cnt * (res * res) / area, rtol=1e-12, atol=0)
    assert want.sum() > 0
    assert np.abs(cnt - want).sum() <= 2 * ties, (np.abs(cnt - want).sum(), ties)


@pytest.mark.gpu
def test_centres_outside_the_mollweide_ellipse_are_not_counted():
    """A shape given in ESRI:54009 that reaches past the ellipse: its centres there are eligible in
    the fine mask and count for no cell of a 4326 cutout."""
    cut = ab.Cutout(data=syn.make_dataset(24, 20, 2, x0=174.125, y0=78.125, kinds=()))
    ex_, ey_ = proj.mollweide_forward(179.0, 83.0)
    edge_x = float(proj.mollweide_forward(180.0, 83.0)[0])
    shape = box(float(ex_) - 2e5, float(ey_) - 1e5, edge_x + 3e5, float(ey_) + 2e5)
    res = 2000.0
    ex = gis.ExclusionContainer(MOLL, res=res)
    m, tr = gis.shape_availability(shape, ex)
    cx = tr[2] + (np.arange(m.shape[1]) + 0.5) * res
    cy = tr[5] - (np.arange(m.shape[0]) + 0.5) * res
    X, Y = np.meshgrid(cx, cy)
    outside = (X / (2 * np.sqrt(2) * R)) ** 2 + (Y / (np.sqrt(2) * R)) ** 2 > 1 + 1e-9
    assert outside.any() and m[outside].any()
    A = cut.availabilitymatrix(InCrs([shape], MOLL), ex)
    want, ties = _oracle_counts(cut, [shape], MOLL, res, [], [])
    x, y = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    xlo, ylo = x - cut.dx / 2, y - cut.dy / 2
    area = proj.mollweide_cell_area(xlo[None], xlo[None] + cut.dx, ylo[:, None], ylo[:, None] + cut.dy)
    cnt = np.rint(np.asarray(A.values) * area / res ** 2).astype(np.int64)
    assert np.abs(cnt - want).sum() <= 2 * ties
    assert 0 < cnt.sum() <= m[~outside].sum()


# ---------------------------------------------------------------- GPU: banded windows
def _budget_for(bands, shape, crs, res, halo=0):
    """A band budget that splits the window of ``shape`` into at least ``bands`` bands."""
    v = np.concatenate([np.asarray(r, float) for r, _ in gis.geometry_rings(shape)]) if isinstance(shape, dict) \
        else np.asarray(shape, float)
    _, (ny, nx) = gis.padded_transform_and_shape((v[:, 0].min(), v[:, 1].min(), v[:, 0].max(), v[:, 1].max()), res)
    rows = max(ny // bands - 1, 1)
    assert -(-ny // rows) >= bands
    return availability._Session.PIXEL_BYTES * nx * (rows + 2 * halo)


def _banded(monkeypatch, budget, fn):
    one = fn()
    with monkeypatch.context() as m:
        m.setattr(availability._Session, "BAND_BYTES", budget)
        many = fn()
    return one, many


@pytest.mark.gpu
def test_bands_equal_one_pass_rasters_lines_and_inverted_geometry(monkeypatch):
    crs, res = MOLL, 500.0
    shape = _in(crs, _outline(8.0, 46.5, 9.4, 47.4))
    rng = np.random.default_rng(6)
    lx, ly = proj.laea_forward(8.7, 46.95)
    lc = gis.Raster(rng.integers(0, 30, (1300, 1300)).astype(np.uint8),
                    (100.0, 0, float(lx) - 6.5e4, 0, -100.0, float(ly) + 6.5e4), 3035)  # cross-CRS
    mx, my = proj.mollweide_forward(8.7, 46.95)
    own = gis.Raster((rng.random((260, 260)) < 0.02).astype(np.uint8),
                     (500.0, 0, float(mx) - 6.5e4, 0, -500.0, float(my) + 6.5e4), MOLL)
    line = InCrs([{"type": "LineString", "coordinates": [[7.9, 46.6], [8.8, 47.3], [9.5, 46.7]]}], 4326)
    inv = InCrs([{"type": "Polygon", "coordinates": [_outline(8.2, 46.6, 9.2, 47.3, 4).tolist()]}], 4326)
    ex = gis.ExclusionContainer(crs, res)
    ex.add_raster(lc, codes=[1, 2, 3, 4])
    ex.add_raster(own, buffer=1900)  # k = 4 rows of halo across every band border
    ex.add_geometry(line, buffer=800)
    ex.add_geometry(inv, invert=True)
    budget = _budget_for(6, shape, crs, res, halo=4)
    one, many = _banded(monkeypatch, budget, lambda: gis.shape_availability(shape, ex))
    assert np.array_equal(one[0], many[0]) and tuple(one[1]) == tuple(many[1])
    assert one[0].any() and not one[0].all()
    cut = ab.Cutout(data=syn.make_dataset(8, 6, 2, x0=8.125, y0=46.625, kinds=()))
    shapes = InCrs([shape], crs)
    one, many = _banded(monkeypatch, budget, lambda: np.asarray(cut.availabilitymatrix(shapes, ex).values))
    assert np.array_equal(one, many) and one.sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("crs", [MOLL, 3857])
def test_bands_equal_one_pass_antimeridian_split_shape(monkeypatch, crs):
    """A shape in two parts at -180 and +180: its window spans the whole map width."""
    parts = [_outline(178.5, 64.0, 180.0, 66.0, 8), _outline(-180.0, 64.5, -178.0, 66.5, 8)]
    shape = {"type": "MultiPolygon", "coordinates": [[_in(crs, p).tolist()] for p in parts]}
    res = 20000.0
    t, shp = gis.padded_transform_and_shape((-180.0, 63.0, 180.0, 67.0), 0.1)
    ex = gis.ExclusionContainer(crs, res)
    ex.add_raster(gis.Raster(np.random.default_rng(7).integers(0, 4, shp).astype(np.uint8), t, 4326), codes=[0],
                  buffer=25000)
    budget = _budget_for(5, shape, crs, res, halo=2)
    one, many = _banded(monkeypatch, budget, lambda: gis.shape_availability(shape, ex))
    assert np.array_equal(one[0], many[0]) and one[0].any()
    assert one[0].shape[1] * res > 2 * float(proj.transform(178.5, 66.0, 4326, crs)[0])  # from -180 to +180
    cut = ab.Cutout(data=syn.make_dataset(1440, 12, 2, x0=-179.875, y0=63.125, kinds=()))
    shapes = InCrs([shape], crs)
    one, many = _banded(monkeypatch, budget, lambda: np.asarray(cut.availabilitymatrix(shapes, ex).values))
    assert np.array_equal(one, many) and one.sum() > 0
