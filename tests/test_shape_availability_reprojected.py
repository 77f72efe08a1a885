"""ExclusionContainer.compute_shape_availability with dst_transform / dst_crs / dst_shape (and
gis.shape_availability_reprojected): the eligible share of every cell of any grid.

The reference pads the mask with zeros (pad_extent) and warps it with GDAL's average.  Here each
destination cell takes gis.reproject's two-corner footprint on the padded window, and its value is
exact integer counts of nine pixel classes combined with the footprint's weights in float64, left to
right.  The references below restate that:

* ``reprojected_exact``: the nine counts from integer 2-D prefix sums of the mask, then the same
  float64 expression in NumPy, so the GPU must match it bit for bit given the same corners;
* ``reprojected_slow``: the window padded with zeros and warped cell by cell with
  oracle/reproject_oracle.py (average), which must agree to 1e-12.

Across CRSs the device projects corners with its own sin / log, which may differ from NumPy's in the
last bits, so the GPU comparison takes the corners the kernels use (``_Session.average_corners``) and
checks them against ``proj.transform`` to 1e-6 pixel separately.  Within one CRS the corners are the
same arithmetic on both sides."""

import ctypes

import numpy as np
import pytest

import atlite_b200 as ab
from atlite_b200 import _lib, availability, gis, proj
from atlite_b200 import synthetic as syn

MOLL = "ESRI:54009"
CRSS = (4326, 3035, 3857, MOLL)
PAIRS = [(a, b) for a in CRSS for b in CRSS]
RES = {4326: 2.0 ** -10, 3035: 100.0, 3857: 128.0, MOLL: 100.0}  # container pixel sizes


# ---------------------------------------------------------------- references
def reference_pad(window_t, crs, dst_t, dst_crs):
    """The reference's pad_extent (gis.py:233-260), restated: the first pixel's bounds T (0, 0) ..
    T (1, 1) through rasterio's transform_bounds (corners and 21 points between them on each edge),
    covered_res their smaller side, pad = int(dst_transform[0] // covered_res * 1.1)."""
    a, _, c, _, e, f = window_t
    left, top, right, bottom = c, f, c + a, f + e
    pts = []
    for (x0, y0), (x1, y1) in [((left, bottom), (right, bottom)), ((right, bottom), (right, top)),
                               ((right, top), (left, top)), ((left, top), (left, bottom))]:
        for k in range(23):
            pts.append((x0 + (x1 - x0) * k / 22, y0 + (y1 - y0) * k / 22))
    px, py = proj.transform(np.array([p[0] for p in pts]), np.array([p[1] for p in pts]), crs, dst_crs)
    covered = (px.min(), py.min(), px.max(), py.max())
    covered_res = min(abs(covered[2] - covered[0]), abs(covered[3] - covered[1]))
    return int(dst_t[0] // covered_res * 1.1)


def lattice_uv(L, crs, dst_t, dst_crs, dst_shape):
    """(ny + 1, nx + 1, 2) window pixel coordinates of the destination lattice points (col, row)."""
    left, top, nx, ny, res = L
    a, _, c, _, e, f = (float(v) for v in tuple(dst_t)[:6])
    jj = np.arange(dst_shape[1] + 1, dtype=np.float64)[None, :]
    ii = np.arange(dst_shape[0] + 1, dtype=np.float64)[:, None]
    x, y = np.broadcast_arrays(c + jj * a, f + ii * e)
    px, py = proj.transform(x, y, dst_crs, crs)
    return np.stack([(px - left) / res, (py - top) / -res], axis=-1)


def _spans(t0, t1, lo_clip, hi_clip):
    lo = np.clip(np.floor(t0 + 1e-10), lo_clip, hi_clip)
    hi = np.clip(np.ceil(t1 - 1e-10), lo_clip, hi_clip)
    return lo, hi, np.fmin(lo + 1.0, t1) - np.fmax(lo, t0), np.fmin(hi, t1) - np.fmax(hi - 1.0, t0)


def _classes(lo, hi, n):
    """(start, stop) of the first, interior and last pixels of each span within [0, n)."""
    two = hi - lo >= 2
    rng = [(lo, lo + 1), (lo + 1, hi - 1), (np.where(two, hi - 1, 0), np.where(two, hi, 0))]
    return [(np.clip(s, 0, n).astype(np.int64), np.clip(np.maximum(t, s), 0, n).astype(np.int64)) for s, t in rng]


def reprojected_exact(eligible, L, crs, dst_t, dst_crs, dst_shape, uv=None):
    """(dst_shape) float64: the window ``eligible`` (L = left, top, nx, ny, res in ``crs``), padded
    by the reference's pad, averaged over each cell's box (corners from ``uv``, default
    ``lattice_uv``) from integer prefix-sum counts; 0 for an empty box or a corner without image."""
    left, top, nx, ny, res = L
    E = np.asarray(eligible, dtype=bool)
    assert E.shape == (ny, nx)
    pad = max(reference_pad((res, 0.0, left, 0.0, -res, top), crs, dst_t, dst_crs), 0)
    if uv is None:
        uv = lattice_uv(L, crs, dst_t, dst_crs, dst_shape)
    P = np.zeros((ny + 1, nx + 1), dtype=np.int64)
    np.cumsum(np.cumsum(E, axis=0, dtype=np.int64), axis=1, out=P[1:, 1:])
    a, b = uv[:-1, :-1], uv[1:, 1:]
    ok = np.isfinite(a).all(-1) & np.isfinite(b).all(-1)
    with np.errstate(invalid="ignore"):
        cx = _spans(np.fmin(a[..., 0], b[..., 0]), np.fmax(a[..., 0], b[..., 0]), -pad, nx + pad)
        cy = _spans(np.fmin(a[..., 1], b[..., 1]), np.fmax(a[..., 1], b[..., 1]), -pad, ny + pad)
        ok &= (cx[1] > cx[0]) & (cy[1] > cy[0])
    cx = [np.where(ok, v, 1.0) for v in cx]
    cy = [np.where(ok, v, 1.0) for v in cy]
    R, K = _classes(cy[0], cy[1], ny), _classes(cx[0], cx[1], nx)

    def count(r, k):
        (r0, r1), (c0, c1) = r, k
        return (P[r1, c1] - P[r0, c1] - P[r1, c0] + P[r0, c0]).astype(np.float64)

    S = [(cx[2] * count(R[q], K[0]) + count(R[q], K[1])) + cx[3] * count(R[q], K[2]) for q in range(3)]
    num = (cy[2] * S[0] + S[1]) + cy[3] * S[2]
    mx, my = cx[1] - cx[0], cy[1] - cy[0]
    Wx = np.where(mx == 1, cx[2], (cx[2] + cx[3]) + (mx - 2))
    Wy = np.where(my == 1, cy[2], (cy[2] + cy[3]) + (my - 2))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(ok, num / (Wy * Wx), 0.0)


def reprojected_slow(eligible, L, crs, dst_t, dst_crs, dst_shape):
    """The window padded with zeros, then reproject_oracle's cell-by-cell average."""
    import reproject_oracle as RO

    left, top, nx, ny, res = L
    pad = max(reference_pad((res, 0.0, left, 0.0, -res, top), crs, dst_t, dst_crs), 0)
    E = np.pad(np.asarray(eligible, dtype=np.float64), pad)
    t = (res, 0.0, left - pad * res, 0.0, -res, top + pad * res)
    return np.nan_to_num(RO.reproject(E, t, crs, dst_t, dst_crs, dst_shape, resampling=5), nan=0.0)


# ---------------------------------------------------------------- geometry of the cases
def _window(crs, nx, ny, lon=10.0, lat=50.0):
    """L = (left, top, nx, ny, res) of a window near (lon, lat), on the container lattice."""
    res = RES[crs]
    x, y = proj.transform(np.float64(lon), np.float64(lat), 4326, crs)
    left, top = np.floor(float(x) / res) * res, np.floor(float(y) / res) * res
    return left, top, nx, ny, res


def _dst_grid(L, crs, dst_crs, cells, margin, south_up):
    """A grid in dst_crs over the window's bounds, about ``cells`` cells across it plus ``margin``
    cells around it."""
    left, top, nx, ny, res = L
    t = np.linspace(0.0, 1.0, 33)
    xs = np.r_[left + nx * res * t, np.full_like(t, left + nx * res), left + nx * res * t, np.full_like(t, left)]
    ys = np.r_[np.full_like(t, top), top - ny * res * t, np.full_like(t, top - ny * res), top - ny * res * t]
    px, py = proj.transform(xs, ys, crs, dst_crs)
    d = max(px.max() - px.min(), py.max() - py.min()) / cells
    gnx = int(np.ceil((px.max() - px.min()) / d)) + 2 * margin
    gny = int(np.ceil((py.max() - py.min()) / d)) + 2 * margin
    x0, y0, y1 = px.min() - margin * d, py.min() - margin * d, py.min() - margin * d + gny * d
    t = (d, 0.0, x0, 0.0, d, y0) if south_up else (d, 0.0, x0, 0.0, -d, y1)
    return t, (gny, gnx)


# ---------------------------------------------------------------- CPU
def test_argument_errors_before_any_device_work():
    ex = gis.ExclusionContainer(3035, 100)
    shape = np.array([[4e6, 3e6], [4.01e6, 3e6], [4.01e6, 3.01e6], [4e6, 3.01e6]])
    t = (0.25, 0.0, 0.0, 0.0, -0.25, 60.0)
    for kw in (dict(dst_crs=4326), dict(dst_transform=t), dict(dst_shape=(4, 4)),
               dict(dst_transform=t, dst_crs=4326), dict(dst_crs=4326, dst_shape=(4, 4))):
        with pytest.raises(NotImplementedError, match="together.*availabilitymatrix"):
            ex.compute_shape_availability(shape, **kw)
    with pytest.raises(NotImplementedError, match="not supported"):
        ex.compute_shape_availability(shape, t, 32632, (4, 4))
    for bad in ((0, 4), (4,), (4, 4, 1), (2.5, 4), (True, 4), "44", 4, (-1, 3), None):
        if bad is None:
            continue
        with pytest.raises(ValueError, match="dst_shape"):
            ex.compute_shape_availability(shape, t, 4326, bad)
    with pytest.raises(ValueError, match="axis-aligned"):
        ex.compute_shape_availability(shape, (0.25, 0.1, 0.0, 0.0, -0.25, 60.0), 4326, (4, 4))
    with pytest.raises(ValueError, match="needs dst_transform"):
        gis.shape_availability_reprojected(shape, ex, t, None, (4, 4))


@pytest.mark.parametrize("side", ["from_", "to"])
def test_average_entry_points_refuse_unknown_crs_before_device_work(side):
    """The descriptors are otherwise valid and the pointers are never touched: the CRS check comes
    first, on the host."""
    lib = _lib.load()
    P = proj.device_projection(4326, 3035)
    getattr(P, side).kind = 7
    A = _lib.AvailAverage(win=_lib.Lattice(4e6, 100.0, 3e6, -100.0, 8, 8),
                          dst=_lib.Lattice(0.0, 0.25, 60.0, -0.25, 4, 4), proj=P, pad=2,
                          row0=0, col0=0, row1=4, col1=4, tile_y=8, tile_x=32)
    rect = (ctypes.c_int32 * 4)()
    for rc in (lib.atl_avail_average_rect(0, ctypes.byref(A), 8, rect, None),
               lib.atl_avail_average_counts(0, ctypes.byref(A), 8, 0, 8, 8, None),
               lib.atl_avail_average_finalize(0, ctypes.byref(A), 8, 8, None),
               lib.atl_avail_average_corners(0, ctypes.byref(A), 8, None)):
        assert rc == -1  # ATL_ERR_INVALID
        assert b"unknown CRS" in lib.atl_last_error()


@pytest.mark.parametrize("crs,dst_crs", PAIRS)
def test_pad_rule_matches_the_reference_formula(crs, dst_crs):
    for lon, lat in ((10.0, 50.0), (-20.0, 70.0), (30.0, 36.0)):
        L = _window(crs, 10, 10, lon, lat)
        wt = (L[4], 0.0, L[0], 0.0, -L[4], L[1])
        for dst_a in ({4326: (0.25, 0.1, 1.0), 3035: (1000.0, 10000.0, 25000.0)}.get(dst_crs, (1000.0, 27000.0))):
            want = reference_pad(wt, crs, (dst_a, 0, 0, 0, -dst_a, 0), dst_crs)
            assert availability.reprojection_pad(wt, crs, dst_a, dst_crs) == want, (lon, lat, dst_a)
    # within one CRS the pad is the destination cell in pixels, plus a tenth
    if crs == dst_crs:
        assert availability.reprojection_pad(wt, crs, 10 * L[4], crs) == 11


@pytest.mark.parametrize("south_up", [False, True])
@pytest.mark.parametrize("crs,dst_crs", PAIRS)
def test_exact_reference_matches_padded_reproject_oracle(crs, dst_crs, south_up):
    rng = np.random.default_rng(abs(hash((str(crs), str(dst_crs), south_up))) % 2 ** 32)
    L = _window(crs, 37, 29)
    E = rng.random((29, 37)) < 0.6
    for cells, margin in ((5, 2), (60, 3)):  # boxes of several pixels, and of one pixel or less
        dt, dshape = _dst_grid(L, crs, dst_crs, cells, margin, south_up)
        if cells == 60:  # a corner of the grid only: the slow oracle walks every cell in Python
            dshape = (min(dshape[0], 20), min(dshape[1], 20))
        want = reprojected_slow(E, L, crs, dt, dst_crs, dshape)
        got = reprojected_exact(E, L, crs, dt, dst_crs, dshape)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
        assert (got > 0).any() and (got == 0).any()


# ---------------------------------------------------------------- GPU
def _container(crs, L, exclusions):
    left, top, nx, ny, res = L
    ex = gis.ExclusionContainer(crs, res)
    w, h = nx * res, ny * res
    shape = np.array([[left + 0.1 * w, top - 0.95 * h], [left + 0.9 * w, top - 0.85 * h], [left + 0.6 * w, top - 0.5 * h],
                      [left + 0.95 * w, top - 0.1 * h], [left + 0.05 * w, top - 0.05 * h]])
    rng = np.random.default_rng(3)
    if "raster" in exclusions or "inverted" in exclusions:
        codes = rng.integers(0, 10, (ny // 2 + 4, nx // 2 + 4)).astype(np.uint8)
        r = gis.Raster(codes, (2 * res, 0.0, left - 4 * res, 0.0, -2 * res, top + 4 * res), crs)
        if "raster" in exclusions:
            ex.add_raster(r, codes=[1, 2], buffer=2 * res)
        if "inverted" in exclusions:
            ex.add_raster(r, codes=[0, 3, 4, 5, 6, 7], invert=True)
    if "line" in exclusions:
        ex.add_geometry([{"type": "LineString", "coordinates": [[left, top - 0.3 * h], [left + w, top - 0.7 * h]]}],
                        buffer=3 * res)
    return ex, shape


def _run(ex, shape, crs, dst_t, dst_crs, dst_shape):
    """(GPU values, host reference from the kernels' corners, the mask's L, the device corners)."""
    mask, t = ex.compute_shape_availability(shape)
    a, _, c, _, e, f = t
    L = (c, f, mask.shape[1], mask.shape[0], a)
    got, gt = ex.compute_shape_availability(shape, dst_t, dst_crs, dst_shape)
    assert gt == dst_t and got.shape == tuple(dst_shape) and got.dtype == np.float64
    with availability._Session(ex) as s:
        parts = availability._parts(shape, crs, proj.epsg(crs), polygonal=True)
        uv = s.average_corners(parts, availability._dst_lattice(dst_t, dst_crs, dst_shape), dst_crs)
    want = reprojected_exact(mask, L, crs, dst_t, dst_crs, dst_shape, uv=uv)
    return got, want, L, uv


def _check_corners(uv, L, crs, dst_t, dst_crs, dst_shape):
    host = lattice_uv(L, crs, dst_t, dst_crs, dst_shape)
    both = np.isfinite(uv) & np.isfinite(host)
    assert both.sum() >= 0.9 * np.isfinite(host).sum()
    np.testing.assert_allclose(uv[both], host[both], rtol=0, atol=1e-6)
    if proj.epsg(crs) == proj.epsg(dst_crs):
        assert np.array_equal(uv, host)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", ["coarse", "fine"])
@pytest.mark.parametrize("south_up", [False, True])
@pytest.mark.parametrize("crs,dst_crs", PAIRS)
def test_bitwise_equal_to_exact_reference(crs, dst_crs, south_up, scale):
    L = _window(crs, 240, 200)
    ex, shape = _container(crs, L, ("raster",))
    cells, margin = (8, 2) if scale == "coarse" else (400, 0)
    dt, dshape = _dst_grid(L, crs, dst_crs, cells, margin, south_up)
    got, want, Lm, uv = _run(ex, shape, crs, dt, dst_crs, dshape)
    _check_corners(uv, Lm, crs, dt, dst_crs, dshape)
    assert np.array_equal(got, want), np.abs(got - want).max()
    assert (got > 0).any() and (got == 0).any() and (got < 1).any()
    if scale == "coarse":
        assert (got[:, 0] == 0).all() and (got[-1] == 0).all()  # the margin: padding and empty cells


@pytest.mark.gpu
@pytest.mark.parametrize("exclusions", [("raster",), ("inverted",), ("line",), ("raster", "inverted", "line")])
@pytest.mark.parametrize("south_up", [False, True])
def test_exclusion_kinds(exclusions, south_up):
    L = _window(3035, 300, 260)
    ex, shape = _container(3035, L, exclusions)
    for dst_crs, cells in ((4326, 6), (3035, 40), (MOLL, 500)):
        dt, dshape = _dst_grid(L, 3035, dst_crs, cells, 1, south_up)
        got, want, _, _ = _run(ex, shape, 3035, dt, dst_crs, dshape)
        assert np.array_equal(got, want), (dst_crs, np.abs(got - want).max())
        assert (got > 0).any()


@pytest.mark.gpu
def test_bands_and_repeats_are_bitwise_equal(monkeypatch):
    L = _window(3035, 400, 300)
    ex, shape = _container(3035, L, ("raster", "line"))
    cases = [(_dst_grid(L, 3035, 4326, 7, 2, False), 4326), (_dst_grid(L, 3035, MOLL, 300, 1, True), MOLL)]
    one = [ex.compute_shape_availability(shape, dt, d, ds)[0] for (dt, ds), d in cases]
    again = [ex.compute_shape_availability(shape, dt, d, ds)[0] for (dt, ds), d in cases]
    monkeypatch.setattr(availability._Session, "BAND_BYTES", availability._Session.PIXEL_BYTES * 400 * 90)
    seen = []
    orig = availability._Session.bands

    def bands(self, parts):
        for b in orig(self, parts):
            seen.append(b[2])
            yield b

    monkeypatch.setattr(availability._Session, "bands", bands)
    many = [ex.compute_shape_availability(shape, dt, d, ds)[0] for (dt, ds), d in cases]
    assert len(set(seen)) >= 3
    for a, b, c in zip(one, again, many):
        assert np.array_equal(a, b) and np.array_equal(a, c) and (a > 0).any()


@pytest.mark.gpu
def test_aligned_grid_is_the_pixel_count_and_the_availabilitymatrix():
    res, cell = 100.0, 10000.0
    x0, y0 = 4000000.0, 2900000.0  # the cutout's lower-left corner, on the 100 m lattice
    ds = syn.make_dataset(12, 10, 2, x0=x0 + cell / 2, y0=y0 + cell / 2, dx=cell, dy=cell, kinds=())
    ds.attrs["crs"] = 3035
    cut = ab.Cutout(data=ds)
    shape = np.array([[x0 + 12345.0, y0 + 8765.0], [x0 + 101234.0, y0 + 15432.0], [x0 + 88888.0, y0 + 91234.0],
                      [x0 + 23456.0, y0 + 76543.0]])
    ex = gis.ExclusionContainer(3035, res)
    codes = np.random.default_rng(5).integers(0, 6, (1000, 1200)).astype(np.uint8)
    ex.add_raster(gis.Raster(codes, (res, 0.0, x0, 0.0, -res, y0 + 1000 * res), 3035), codes=[1], buffer=150)
    for t in (cut.transform, cut.transform_r):
        got, _ = ex.compute_shape_availability(shape, t, 3035, (10, 12))
        mask, mt = ex.compute_shape_availability(shape)
        # the eligible pixels of each 100 x 100 block of the grid, from the mask
        i0 = int(round((mt[2] - x0) / res))
        j0 = int(round((y0 + 10 * cell - mt[5]) / res))
        full = np.zeros((1000, 1200), dtype=np.int64)
        full[j0:j0 + mask.shape[0], i0:i0 + mask.shape[1]] = mask
        count = full.reshape(10, 100, 12, 100).sum(axis=(1, 3))  # rows from the top
        want = count / 10000.0
        if t[4] > 0:
            want = want[::-1]
        assert np.array_equal(got, want)
        A = np.asarray(cut.availabilitymatrix([shape], ex).values)[0]  # y ascending
        A = A if t[4] > 0 else A[::-1]
        np.testing.assert_allclose(got, A, rtol=1e-15, atol=0)
        assert (got > 0).sum() > 20


@pytest.mark.gpu
@pytest.mark.parametrize("dst", ["4326_025", "4326_01", "moll_1km"])
def test_production_footprint(dst):
    """About 900 x 800 km at 100 m (7.2e7 pixels) in EPSG:3035 with a land-cover raster."""
    res = 100.0
    left, top = 3900000.0, 3300000.0
    nx, ny = 9000, 8000
    w, h = nx * res, ny * res
    shape = np.array([[left + 0.02 * w, top - 0.98 * h], [left + 0.97 * w, top - 0.9 * h], [left + 0.99 * w, top - 0.3 * h],
                      [left + 0.6 * w, top - 0.45 * h], [left + 0.55 * w, top - 0.02 * h], [left + 0.01 * w, top - 0.1 * h]])
    rng = np.random.default_rng(11)
    lc = rng.integers(0, 40, (ny // 4 + 2, nx // 4 + 2)).astype(np.uint8)
    ex = gis.ExclusionContainer(3035, res)
    ex.add_raster(gis.Raster(lc, (4 * res, 0.0, left - 4 * res, 0.0, -4 * res, top + 4 * res), 3035),
                  codes=list(range(20, 40)), buffer=300)
    if dst == "4326_025":
        dt, dshape = (0.25, 0.0, -12.0, 0.0, 0.25, 35.0), (120, 200)
    elif dst == "4326_01":
        dt, dshape = (0.1, 0.0, -10.0, 0.0, -0.1, 66.0), (300, 400)
    else:
        dt, dshape = (1000.0, 0.0, -500000.0, 0.0, -1000.0, 6800000.0), (1200, 1600)
    dst_crs = MOLL if dst == "moll_1km" else 4326
    got, want, L, uv = _run(ex, shape, 3035, dt, dst_crs, dshape)
    assert L[2] * L[3] > 6e7
    _check_corners(uv, L, 3035, dt, dst_crs, dshape)
    assert np.array_equal(got, want), np.abs(got - want).max()
    assert (got > 0).sum() > 50 and (got == 0).any()
