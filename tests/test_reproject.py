"""gis.reproject: rasters warped between EPSG:4326, 3035, 3857 and ESRI:54009 (rasterio.warp.reproject
with Resampling.average / .nearest).

CPU: argument errors before any device work, the oracle (oracle/reproject_oracle.py) against the
regrid_axis(pad=0) tables within one CRS, constant fields, and the orientation dependence of the
two-corner footprint.  GPU: every supported pair against the oracle in both regimes (boxes summed by
one thread and by a whole CTA), nodata, cells without an image, the same-CRS routing through
k_regrid, determinism, and a GeoTIFF layout end to end through ``Cutout.temperature``.
"""

import numpy as np
import pytest

import reproject_oracle as RO
from atlite_b200 import engine, gis, proj

MOLL = "ESRI:54009"


def _bounds(crs, lon0, lon1, lat0, lat1):
    """(left, bottom, right, top) in ``crs`` of the lon / lat box, from 33 points per edge."""
    t = np.linspace(0.0, 1.0, 33)
    lon = np.concatenate([lon0 + t * (lon1 - lon0), np.full(33, lon1), lon1 - t * (lon1 - lon0), np.full(33, lon0)])
    lat = np.concatenate([np.full(33, lat0), lat0 + t * (lat1 - lat0), np.full(33, lat1), lat1 - t * (lat1 - lat0)])
    x, y = proj.transform(lon, lat, 4326, crs)
    return x.min(), y.min(), x.max(), y.max()


def _grid(crs, box, shape, south_up=False):
    """Transform of a ``shape`` grid over the lon / lat ``box``, north-up or south-up."""
    left, bottom, right, top = _bounds(crs, *box)
    a, e = (right - left) / shape[1], (top - bottom) / shape[0]
    return (a, 0.0, left, 0.0, e, bottom) if south_up else (a, 0.0, left, 0.0, -e, top)


SRC_BOX, DST_BOX = (2.0, 22.0, 40.0, 58.0), (0.0, 24.0, 38.0, 60.0)  # the destination overhangs the source


# ---------------------------------------------------------------- CPU

def _no_device(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("device work before the argument check")

    monkeypatch.setattr(engine, "ReprojectOp", boom)
    monkeypatch.setattr(engine, "RegridOp", boom)


def test_argument_errors(monkeypatch):
    _no_device(monkeypatch)
    v = np.ones((4, 5))
    st, dt = (1.0, 0.0, 0.0, 0.0, -1.0, 4.0), (2.0, 0.0, 0.0, 0.0, -2.0, 4.0)
    ok = dict(src_transform=st, src_crs=4326)
    with pytest.raises(NotImplementedError, match="resampling"):
        gis.reproject(v, dt, 4326, (2, 2), resampling=1, **ok)
    with pytest.raises(NotImplementedError, match="resampling"):
        gis.reproject(v, dt, 4326, (2, 2), resampling=True, **ok)
    with pytest.raises(NotImplementedError):
        gis.reproject(v, dt, 2154, (2, 2), **ok)
    with pytest.raises(NotImplementedError):
        gis.reproject(v, dt, 4326, (2, 2), src_transform=st, src_crs=54009)
    with pytest.raises(TypeError, match="float32 and float64"):
        gis.reproject(v.astype(np.int32), dt, 4326, (2, 2), **ok)
    with pytest.raises(ValueError, match="axis-aligned"):
        gis.reproject(v, (2.0, 0.5, 0.0, 0.0, -2.0, 4.0), 4326, (2, 2), **ok)
    with pytest.raises(ValueError, match="axis-aligned"):
        gis.reproject(v, dt, 4326, (2, 2), src_transform=(0.0, 0.0, 0.0, 0.0, -1.0, 4.0), src_crs=4326)
    with pytest.raises(ValueError, match="src_transform and src_crs"):
        gis.reproject(v, dt, 4326, (2, 2), src_crs=4326)
    with pytest.raises(ValueError, match="dst_shape"):
        gis.reproject(v, dt, 4326, (2, -1), **ok)
    with pytest.raises(ValueError, match="dst_shape"):
        gis.reproject(v, dt, 4326, (2, 2, 2), **ok)
    with pytest.raises(ValueError, match=r"\(\.\.\., ny, nx\)"):
        gis.reproject(np.ones(5), dt, 4326, (2, 2), **ok)
    with pytest.raises(TypeError, match="dst_nodata"):
        gis.reproject(v, dt, 4326, (2, 2), dst_nodata="x", **ok)
    r = gis.Raster(v, st, 4326, nodata=-1.0)
    for kw in (dict(src_crs=3035), dict(src_transform=dt), dict(src_nodata=0.0)):
        with pytest.raises(ValueError, match="contradicts"):
            gis.reproject(r, dt, 4326, (2, 2), **kw)
    with pytest.raises(NotImplementedError, match="resampling"):  # agreeing keywords pass the check
        gis.reproject(r, dt, 4326, (2, 2), src_crs="EPSG:4326", src_transform=st, src_nodata=-1.0, resampling=2)


def _host_tables(values, st, src_shape, dt, dst_shape, nearest=False):
    """The same-CRS tables applied on the host: row x-sums, then the rows."""
    (yf, yc, yw), (xf, xc, xw) = gis._same_crs_tables(st, src_shape, dt, dst_shape, nearest)
    out = np.full(dst_shape, np.nan)
    for i in range(dst_shape[0]):
        for j in range(dst_shape[1]):
            s = w = 0.0
            for k in range(yc[i]):
                row = values[yf[i] + k, xf[j]:xf[j] + xc[j]]
                ok = ~np.isnan(row)
                s += yw[i, k] * np.sum(xw[j, :xc[j]] * np.where(ok, row, 0.0))
                w += yw[i, k] * np.sum(xw[j, :xc[j]] * ok)
            if w > 0:
                out[i, j] = s / w
    return out


@pytest.mark.parametrize("src_sign", [(1, -1), (1, 1), (-1, -1)])
@pytest.mark.parametrize("dst_sign", [(1, -1), (1, 1), (-1, 1)])
@pytest.mark.parametrize("resampling", [5, 0])
def test_same_crs_oracle_equals_regrid_tables(src_sign, dst_sign, resampling):
    rng = np.random.default_rng(1)
    v = rng.uniform(0.5, 1.5, (24, 20))
    v[3, 4] = np.nan
    sa, se = 0.25 * src_sign[0], 0.25 * src_sign[1]
    st = (sa, 0.0, 4.0 if sa > 0 else 9.0, 0.0, se, 50.0 if se < 0 else 44.0)
    da, de = 0.75 * dst_sign[0], 0.625 * dst_sign[1]
    off = 0.1 if resampling == 0 else 0.0  # nearest: centres off the (dyadic) pixel edges
    dt = (da, 0.0, (4.125 if da > 0 else 9.375) + off, 0.0, de, (43.5 if de > 0 else 50.5) + off)
    got = _host_tables(v, st, v.shape, dt, (12, 11), resampling == 0)
    want = RO.reproject(v, st, 3035, dt, 3035, (12, 11), resampling)
    assert not (RO.centre_edge_distance(st, 3035, dt, 3035, (12, 11)) < 1e-9).any() or resampling == 5
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.isnan(want).any() and (~np.isnan(want)).sum() > 40
    np.testing.assert_allclose(got, want, rtol=1e-15, atol=0)


@pytest.mark.parametrize("src,dst", [(3035, 4326), (4326, MOLL), (4326, 3857)])
def test_constant_field(src, dst):
    st = _grid(src, SRC_BOX, (30, 36))
    dt = _grid(dst, DST_BOX, (7, 9))
    v = np.full((30, 36), 0.7)
    v[:4, :5] = np.nan
    got = RO.reproject(v, st, src, dt, dst, (7, 9), 5)
    ok = ~np.isnan(got)
    assert ok.sum() > 20
    np.testing.assert_allclose(got[ok], 0.7, rtol=1e-14)


def _flip_rows(t, ny):
    a, b, c, d, e, f = t
    return (a, b, c, d, -e, f + ny * e)


@pytest.mark.parametrize("src,dst", [(3035, 4326), (4326, 3035), (MOLL, 4326)])
def test_orientation(src, dst):
    """The footprint spans two corners, so north-up and south-up destinations of the same cells
    differ across CRSs; within one CRS they are the same boxes."""
    rng = np.random.default_rng(2)
    st = _grid(src, SRC_BOX, (40, 44))
    v = rng.uniform(0.5, 1.5, (40, 44))
    north = _grid(dst, DST_BOX, (6, 8))
    south = _flip_rows(north, 6)
    a = RO.reproject(v, st, src, north, dst, (6, 8), 5)
    b = RO.reproject(v, st, src, south, dst, (6, 8), 5)[::-1]
    assert np.nanmax(np.abs(a - b)) > 1e-4
    north = _grid(src, DST_BOX, (6, 8))
    a = RO.reproject(v, st, src, north, src, (6, 8), 5)
    b = RO.reproject(v, st, src, _flip_rows(north, 6), src, (6, 8), 5)[::-1]
    np.testing.assert_allclose(a, b, rtol=1e-13)


# ---------------------------------------------------------------- GPU

PAIRS = [(4326, 3035), (3035, 4326), (4326, 3857), (3857, 4326), (4326, MOLL), (MOLL, 4326), (3035, MOLL),
         (MOLL, 3035)]
REGIMES = {"down": ((60, 72), (9, 11)), "up": ((12, 14), (30, 34))}  # (source, destination) shapes


def _case(src, dst, regime, south_up, lead=(2,), seed=0):
    sshape, dshape = REGIMES[regime]
    rng = np.random.default_rng(seed)
    st = _grid(src, SRC_BOX, sshape)
    dt = _grid(dst, DST_BOX, dshape, south_up)
    return rng.uniform(0.5, 1.5, lead + sshape), st, dt, dshape


def _check(got, want, resampling, st, src, dt, dst, dshape, rtol=1e-9):
    got = got.cpu().numpy() if hasattr(got, "cpu") else got
    assert got.shape == want.shape
    if resampling == 5:
        assert np.array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_allclose(got, want, rtol=rtol, atol=0)
        return
    sure = ~(RO.centre_edge_distance(st, src, dt, dst, dshape) < 1e-9)
    np.testing.assert_array_equal(got[..., sure], want[..., sure])


@pytest.mark.gpu
@pytest.mark.parametrize("south_up", [False, True], ids=["north", "south"])
@pytest.mark.parametrize("resampling", [5, 0], ids=["average", "nearest"])
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_pairs_against_oracle(src, dst, regime, resampling, south_up):
    import torch

    v, st, dt, dshape = _case(src, dst, regime, south_up)
    want = RO.reproject(v, st, src, dt, dst, dshape, resampling)
    assert (~np.isnan(want)).sum() > 0.3 * want.size
    got, t = gis.reproject(torch.from_numpy(v).cuda(), dt, dst, dshape, src_transform=st, src_crs=src,
                           resampling=resampling)
    assert got.is_cuda and got.dtype == torch.float64 and t == dt
    _check(got, want, resampling, st, src, dt, dst, dshape)


def _box_pixels(src, dst, regime):
    """Source pixels of every destination cell's two-corner box in a regime."""
    _, st, dt, (ny, nx) = _case(src, dst, regime, False, lead=())
    jj, ii = np.meshgrid(np.arange(nx + 1), np.arange(ny + 1))
    x, y = proj.transform(dt[2] + jj * dt[0], dt[5] + ii * dt[4], dst, src)
    u, v = (x - st[2]) / st[0], (y - st[5]) / st[4]
    w = np.ceil(np.maximum(u[:-1, :-1], u[1:, 1:])) - np.floor(np.minimum(u[:-1, :-1], u[1:, 1:]))
    h = np.ceil(np.maximum(v[:-1, :-1], v[1:, 1:])) - np.floor(np.minimum(v[:-1, :-1], v[1:, 1:]))
    return w * h


@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_regimes_take_both_paths(src, dst):
    """"down" boxes exceed the 32 pixels one thread sums (a CTA sums them), "up" boxes do not."""
    assert np.median(_box_pixels(src, dst, "down")) > 32
    assert np.nanmax(_box_pixels(src, dst, "up")) <= 32


@pytest.mark.gpu
@pytest.mark.parametrize("resampling", [5, 0])
def test_float32_batch_and_host(resampling):
    v, st, dt, dshape = _case(4326, 3035, "down", True, lead=(2, 3), seed=4)
    v32 = v.astype(np.float32)
    want = RO.reproject(v32, st, 4326, dt, 3035, dshape, resampling)
    got, _ = gis.reproject(v32, dt, 3035, dshape, src_transform=st, src_crs=4326, resampling=resampling)
    assert isinstance(got, np.ndarray) and got.dtype == np.float32 and got.shape == (2, 3) + dshape
    _check(got, want, resampling, st, 4326, dt, 3035, dshape, rtol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("resampling", [5, 0])
@pytest.mark.parametrize("src,dst", [(4326, 3035), (3035, 3035)], ids=["cross", "same"])
def test_nodata(src, dst, resampling):
    v, st, dt, dshape = _case(src, dst, "down", False, lead=(), seed=5)
    v[::7, ::5] = np.nan
    v[1::6, ::4] = -9999.0
    v[20:45, 20:40] = -9999.0  # whole cells without a valid pixel
    r = gis.Raster(v, st, src, nodata=-9999.0)
    for dst_nodata, fill in ((None, -9999.0), (np.nan, np.nan), (-1.0, -1.0)):
        want = RO.reproject(v, st, src, dt, dst, dshape, resampling, -9999.0, dst_nodata)
        got, _ = gis.reproject(r, dt, dst, dshape, resampling=resampling, dst_nodata=dst_nodata)
        assert (want == fill).any() or np.isnan(fill)
        assert not (want == -9999.0).any() or fill == -9999.0
        if np.isnan(fill):
            assert np.isnan(got).sum() > np.isnan(RO.reproject(np.ones_like(v), st, src, dt, dst, dshape)).sum()
        _check(got, want, resampling, st, src, dt, dst, dshape)
    got, _ = gis.reproject(v, dt, dst, dshape, src_transform=st, src_crs=src, resampling=resampling)
    assert (got == -9999.0).any()  # without src_nodata the value is data


@pytest.mark.gpu
@pytest.mark.parametrize("resampling", [5, 0])
@pytest.mark.parametrize("dst,box", [(MOLL, (-2.0e7, -1.0e7, 2.0e7, 1.0e7)), (3857, (-2.2e7, -1.2e7, 2.2e7, 1.2e7))],
                         ids=["mollweide-ellipse", "mercator-map"])
def test_cells_without_an_image(dst, box, resampling):
    rng = np.random.default_rng(6)
    v = rng.uniform(0.5, 1.5, (36, 72))
    st = (5.0, 0.0, -180.0, 0.0, -5.0, 90.0)
    left, bottom, right, top = box
    dshape = (12, 22)
    dt = ((right - left) / dshape[1], 0.0, left, 0.0, -(top - bottom) / dshape[0], top)
    want = RO.reproject(v, st, 4326, dt, dst, dshape, resampling, dst_nodata=-1.0)
    assert (want == -1.0).sum() >= 4 and (want != -1.0).sum() > want.size // 2
    got, _ = gis.reproject(v, dt, dst, dshape, src_transform=st, src_crs=4326, resampling=resampling,
                           dst_nodata=-1.0)
    _check(got, want, resampling, st, 4326, dt, dst, dshape)


def _profile_kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


@pytest.mark.gpu
@pytest.mark.parametrize("resampling", [5, 0])
@pytest.mark.parametrize("south_up", [False, True])
def test_same_crs_runs_k_regrid(resampling, south_up):
    import torch

    v, st, dt, dshape = _case(3035, 3035, "down", south_up, lead=(3,), seed=7)
    v[:, ::9, ::7] = np.nan
    t = torch.from_numpy(v).cuda()
    got = {}
    names = _profile_kernels(lambda: got.update(r=gis.reproject(t, dt, 3035, dshape, src_transform=st, src_crs=3035,
                                                              resampling=resampling)[0]))
    assert any("k_regrid" in n for n in names) and not any("k_reproject" in n for n in names), names
    ident = engine.ReprojectOp((st, v.shape[1:], 3035), (dt, dshape, 3035), resampling)(t)
    a, b = got["r"].cpu().numpy(), ident.cpu().numpy()
    if resampling == 5:
        assert np.array_equal(np.isnan(a), np.isnan(b))
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=0)
    else:
        sure = ~(RO.centre_edge_distance(st, 3035, dt, 3035, dshape) < 1e-9)
        np.testing.assert_array_equal(a[..., sure], b[..., sure])
    names = _profile_kernels(lambda: gis.reproject(t, dt, 4326, dshape, src_transform=st, src_crs=3035,
                                                   resampling=resampling))
    assert any("k_reproject" in n for n in names) and not any("k_regrid" in n for n in names), names


@pytest.mark.gpu
@pytest.mark.parametrize("resampling", [5, 0])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_deterministic(regime, resampling, monkeypatch):
    import torch

    v, st, dt, dshape = _case(3035, 4326, regime, True, lead=(5,), seed=8)
    kw = dict(src_transform=st, src_crs=3035, resampling=resampling)
    dev = gis.reproject(torch.from_numpy(v).cuda(), dt, 4326, dshape, **kw)[0].cpu().numpy()
    host = gis.reproject(v, dt, 4326, dshape, **kw)[0]
    again = gis.reproject(v, dt, 4326, dshape, **kw)[0]
    assert np.array_equal(dev, host, equal_nan=True) and np.array_equal(host, again, equal_nan=True)
    for b in range(5):
        one = gis.reproject(v[b], dt, 4326, dshape, **kw)[0]
        assert np.array_equal(one, host[b], equal_nan=True)
    monkeypatch.setattr(engine.ReprojectOp, "HOST_SLAB_BYTES", 1)  # one entry per slab
    assert np.array_equal(gis.reproject(v, dt, 4326, dshape, **kw)[0], host, equal_nan=True)
    for tile in ((1, 1), (2, 4), (8, 32)):
        op = engine.ReprojectOp((st, v.shape[1:], 3035), (dt, dshape, 4326), resampling, tile=tile)
        assert np.array_equal(op(v), host, equal_nan=True), tile


@pytest.mark.gpu
def test_geotiff_layout_end_to_end(tmp_path):
    """A float32 EPSG:3035 population raster, written as a GeoTIFF and read with geotiff.read, warped
    onto a cutout's grid, normalised, and used as the layout of Cutout.temperature."""
    from conftest import assert_parity, oracle_ds
    from test_geotiff import write_tiff

    import atlite_oracle as O
    import atlite_b200 as ab
    from atlite_b200 import geotiff, synthetic as syn
    from atlite_b200.labelled import DataArray

    ds = syn.make_dataset(16, 12, 24, x0=5.0, y0=45.0)
    cut = ab.Cutout(data=ds)
    left, bottom, right, top = _bounds(3035, 4.5, 9.5, 44.5, 48.5)
    res = 5000.0
    x0, y0 = np.floor(left / res) * res, np.ceil(top / res) * res
    shape = (int(np.ceil((y0 - bottom) / res)), int(np.ceil((x0 - right) / -res)))
    pop = np.random.default_rng(9).gamma(2.0, 50.0, shape).astype(np.float32)
    path = write_tiff(str(tmp_path / "pop.tif"), pop, epsg=3035, scale=res, origin=(x0, y0), block=(16, 0))
    ras = geotiff.read(path)
    lay, t = gis.reproject(ras, cut.transform, cut.crs, cut.shape, resampling=5)
    assert lay.is_cuda and t == cut.transform
    lay = lay.cpu().numpy()
    lay = lay / lay.sum()
    st = (res, 0.0, x0, 0.0, -res, y0)
    want_lay = RO.reproject(pop, st, 3035, tuple(cut.transform)[:6], 4326, cut.shape, 5)
    want_lay = want_lay / want_lay.sum()
    assert not np.isnan(want_lay).any()
    np.testing.assert_allclose(lay, want_lay, rtol=1e-5)
    layout = DataArray(lay, {"y": ds.coords["y"], "x": ds.coords["x"]}, ("y", "x"))
    got = np.asarray(cut.temperature(layout=layout, aggregate_time=None).values)
    want = O.convert_and_aggregate(oracle_ds(ds), O.convert_temperature, layout=want_lay, aggregate_time=None)
    got = got if got.shape == want.shape else got.T
    assert_parity(got, want, capacity=300.0, what="temperature layout", additive=True)
